"""The batched LZ4 frame compressor (swc_lz4_frame_compress_batch, the "lz4_frame_compress" Batch codec) byte for byte against
the CPU restatement of LZ4.compress (oracle/swco_lz4c.py), and every frame back through the "lz4_frame" decode batch: the
option sweep, dictionaries and dictionary IDs, the reference's traps, the stored-block rule, hostile input and output
layouts with capacity fences, slices of the scratch, the block table's capacity, a CUDA-graph capture and the benched shape."""
import ctypes as C
import random

import numpy as np
import pytest

import helpers as H
import lz4c_cases as K

pytestmark = pytest.mark.gpu
OK, OVERFLOW, TRAP, INVALID_ARG, UNSUPPORTED = 0, 1, 2, 4, 6
FLAGS = [dict(independentBlocks=ind, blockChecksums=bc, contentChecksum=cc, contentSize=cs)
         for ind in (True, False) for bc in (False, True) for cc in (False, True) for cs in (False, True)]


@pytest.fixture(scope="module")
def oc():
    import swco_lz4c
    swco_lz4c.lib()
    return swco_lz4c


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


def _bound(n, opts, dict_id=None):
    from swcompression_b200 import LZ4
    return LZ4.max_compressed_size(n, opts.get("blockChecksums", False), opts.get("contentChecksum", True),
                                   opts.get("contentSize", False), opts.get("blockSize", 4 << 20), dict_id)


def _frames(units, opts, dictionary=None, dict_id=None, caps=None, max_blocks=None, scratch_bytes=None):
    """-> (Batch, status, out_len, outputs) of one "lz4_frame_compress" batch; caps default to the exact bound"""
    from swcompression_b200.batch import Batch
    flags = {k: v for k, v in opts.items() if k != "blockSize"}
    if caps is None:
        caps = np.array([_bound(len(u), opts, dict_id) for u in units], dtype=np.uint64)
    b = Batch.from_units("lz4_frame_compress", units, caps, aux=dictionary, dict_id=dict_id, max_blocks=max_blocks,
                         scratch_bytes=scratch_bytes, block_size=opts.get("blockSize"), frame_flags=flags)
    b.run()
    st, ln, used = b.results()
    assert (used == 0).all()
    return b, st, ln, b.outputs()


def _check(oc, units, st, ln, outs, opts, dictionary=None, dict_id=None):
    """every unit against the oracle; the OK ones decoded back through the "lz4_frame" batch"""
    from swcompression_b200.batch import Batch
    good = []
    for i, u in enumerate(units):
        ost, exp, _ = oc.lz4_compress(u, dictionary=dictionary, dictionaryID=dict_id, **opts)
        assert st[i] == ost, (i, len(u), int(st[i]), ost, opts)
        if ost == OK:
            assert ln[i] == len(exp) and outs[i] == exp, (i, len(u), int(ln[i]), len(exp), opts)
            good.append(i)
        else:
            assert ln[i] == 0, i
    if good:
        d = dictionary if dictionary is not None or dict_id is None else b""
        back = Batch.from_units("lz4_frame", [outs[i] for i in good], np.array([max(len(units[i]), 1) for i in good], dtype=np.uint64),
                                aux=d, dict_id=dict_id)
        back.run()
        bst, _, _ = back.results()
        assert (bst == OK).all() and back.outputs() == [units[i] for i in good]
    return good


def _sweep_units(bs):
    text = dict(K.frame_inputs())["text"]
    rng = random.Random(bs)
    units = [d for _, d in K.frame_inputs()] + list(K.STRINGS) + [K.TRICKY]
    for n in (0, 1, bs - 1, bs, bs + 1, 3 * bs):
        tiled = (text * (n // len(text) + 1))[:n]
        if n > 64:                       # a random stretch in the middle: some blocks stored, some not
            k = rng.randrange(n // 2)
            tiled = tiled[:k] + H.random_bytes(rng, min(n - k, 3000)) + tiled[k + 3000:]
        units.append(tiled[:n])
    return units


@pytest.mark.parametrize("bs", K.SWEEP_BLOCK_SIZES)
def test_option_sweep(S, oc, bs):
    """every combination of the four flags, one batch each, over the sweep inputs, the reference strings and lengths around
    the block size"""
    units = _sweep_units(bs)
    for flags in FLAGS:
        opts = dict(flags, blockSize=bs)
        _, st, ln, outs = _frames(units, opts)
        assert len(_check(oc, units, st, ln, outs, opts)) == len(units)


def test_default_options(S, oc):
    """no options at all: the frame of LZ4.compress(data:)"""
    from swcompression_b200.batch import Batch
    units = [d for _, d in K.frame_inputs()] + list(K.STRINGS)
    b = Batch.from_units("lz4_frame_compress", units, np.array([_bound(len(u), {}) for u in units], dtype=np.uint64))
    b.run()
    st, ln, _ = b.results()
    assert b.block_size == 4 << 20
    assert (st == OK).all() and b.outputs() == [oc.lz4_compress(u)[1] for u in units]


def test_dictionaries(S, oc):
    """None, empty, the small fixture, one past 64 KiB and a 4-byte one, in both block modes; dictionary IDs with and without
    a dictionary"""
    text = dict(K.frame_inputs())["text"]
    small = H.fixture("LZ4/lz4_small_dict")
    rng = random.Random(2)
    big = H.random_bytes(rng, 30000) + text[:50000]
    units = [text, text[:5000], text[1000:1100], b"", b"x", text[:65536 * 2 + 17]]
    for d in (None, b"", small, big, text[:4]):
        for ind in (True, False):
            for dict_id in (None, 20000):
                opts = dict(independentBlocks=ind, blockChecksums=True, contentChecksum=True, contentSize=ind, blockSize=65536)
                _, st, ln, outs = _frames(units, opts, d, dict_id)
                assert len(_check(oc, units, st, ln, outs, opts, d, dict_id)) == len(units), (d and len(d), ind, dict_id)


def test_traps(S, oc):
    """1-3 byte dictionaries trap on non-empty units only; dependent blocks of 1-3 bytes trap once there are two of them;
    a block size outside 1 ... 4 MiB is the call's trap and no status is written"""
    units = [b"", b"a", b"abcdefgh", b"abc", K.TRICKY, b""]
    for d in (b"a", b"ab", b"abc"):
        for ind in (True, False):
            opts = dict(FLAGS[3], independentBlocks=ind, blockSize=65536)
            _, st, ln, outs = _frames(units, opts, d)
            assert list(st) == [OK, TRAP, TRAP, TRAP, TRAP, OK]
            _check(oc, units, st, ln, outs, opts, d)
    for bs in (1, 2, 3):
        for ind in (True, False):
            units = [b"", b"a", b"ab", b"abc", b"abcd", b"abcdefgh", K.TRICKY]
            opts = dict(FLAGS[7], independentBlocks=ind, blockSize=bs)
            _, st, ln, outs = _frames(units, opts)
            good = _check(oc, units, st, ln, outs, opts)
            assert len(good) == (len(units) if ind else sum(len(u) <= bs for u in units))
    from swcompression_b200.batch import Batch
    for bs in (0, -5, (4 << 20) + 1):
        b = Batch.from_units("lz4_frame_compress", [b"abcdefgh", b""], 64, block_size=bs)
        with pytest.raises(RuntimeError, match="referenceTrap"):
            b.run()
        st, ln, _ = b.results()
        assert (st == -1).all() and (ln == 0).all()


def test_stored_rule(S, oc):
    """incompressible units are stored, a block whose compressed form is exactly as long stays compressed, and frames mix
    stored and compressed blocks"""
    rng = random.Random(11)
    eq = K.compressible_equal_size()
    text = dict(K.frame_inputs())["text"]
    units = [H.random_bytes(rng, n) for n in (1, 13, 100, 4097, 65536, 300000)] + [eq, eq * 3]
    units.append(b"".join(text[k * 5000:(k + 1) * 5000] if k % 2 else H.random_bytes(rng, 5000) for k in range(12)))
    for ind in (True, False):
        opts = dict(independentBlocks=ind, blockChecksums=True, contentChecksum=True, contentSize=True, blockSize=5000)
        _, st, ln, outs = _frames(units, opts)
        _check(oc, units, st, ln, outs, opts)
        for i in range(6):
            assert ln[i] == _bound(len(units[i]), opts)                   # every block stored
        mark = int.from_bytes(outs[6][15:19], "little")
        assert mark == len(eq) and outs[6][19:19 + len(eq)] != eq          # kept compressed although no shorter
        marks, at = [], 15
        while True:
            m = int.from_bytes(outs[8][at:at + 4], "little")
            if m == 0:
                break
            marks.append(m >> 31)
            at += 4 + (m & 0x7FFFFFFF) + 4
        assert 0 < sum(marks) < len(marks)


def _layout_call(buf, offs, lens, out_off, out_cap, total, opts, max_blocks=0):
    import torch
    from swcompression_b200 import _lib
    n = len(offs)
    d_in, d_off, d_len, d_oo, d_oc = _dev(buf), _dev(offs), _dev(lens), _dev(out_off), _dev(out_cap)
    d_out = torch.full((total,), H.SENTINEL, dtype=torch.uint8, device="cuda")
    d_ln = torch.zeros(n, dtype=torch.int64, device="cuda")
    d_st = torch.full((n,), -1, dtype=torch.int32, device="cuda")
    assert _lib.lib().swc_lz4_frame_compress_batch(
        _p(d_in), _p(d_off), _p(d_len), int(opts["independentBlocks"]), int(opts["blockChecksums"]), int(opts["contentChecksum"]),
        int(opts["contentSize"]), opts["blockSize"], None, 0, 0, 0, _p(d_out), _p(d_oo), _p(d_oc), _p(d_ln), _p(d_st), n,
        max_blocks, None, 0, C.c_void_p(torch.cuda.current_stream().cuda_stream)) == 0
    torch.cuda.synchronize()
    out = d_out.cpu().numpy()
    outs = [bytes(out[int(o):int(o) + int(c)]) for o, c in zip(out_off, out_cap)]
    return d_st.cpu().numpy(), d_ln.cpu().numpy(), outs, H.fence_violations(out, out_off, out_cap)


def test_hostile_layout(S, oc):
    """inputs packed with no friendly bytes around them, outputs at every start residue with capacities exact, 1-15 bytes
    short (overflow with the exact size, sentinels intact) and 1-15 long; the overflowing ones rerun at out_len"""
    rng = random.Random(74)
    text = dict(K.frame_inputs())["text"]
    units = []
    for j in range(300):
        n = rng.choice((0, 1, 7, 100, 1000, 4095, 4096, 4097, 9000, 20000))
        k = rng.randrange(len(text) - n) if n < len(text) else 0
        units.append(text[k:k + n] if j % 4 else H.random_bytes(rng, n))
    for opts in (dict(independentBlocks=False, blockChecksums=True, contentChecksum=True, contentSize=True, blockSize=4096),
                 dict(independentBlocks=True, blockChecksums=False, contentChecksum=False, contentSize=False, blockSize=1024)):
        want = [oc.lz4_compress(u, **opts)[1] for u in units]
        out_off, out_cap, total = H.fenced_layout([len(w) for w in want])
        buf, offs, lens = H.pack_hostile(units, rng)
        st, ln, outs, fence = _layout_call(buf, offs, lens, out_off, out_cap, total, opts)
        assert fence.size == 0, fence[:8]
        for i, w in enumerate(want):
            assert ln[i] == len(w), i
            if out_cap[i] >= len(w):
                assert st[i] == OK and outs[i][:len(w)] == w, i
            else:
                assert st[i] == OVERFLOW, i
        redo = [i for i in range(len(units)) if st[i] == OVERFLOW]
        assert len(redo) > 50
        _, st2, ln2, outs2 = _frames([units[i] for i in redo], opts, caps=ln[redo].astype(np.uint64))
        assert (st2 == OK).all() and outs2 == [want[i] for i in redo]


def _min_scratch(units, opts):
    """the smallest scratch the call takes (one block per slice): below it the call is SWC_ERR_INVALID_ARG"""
    lo, hi = 1, 1 << 30
    while lo < hi:
        mid = (lo + hi) // 2
        try:
            _frames(units, opts, scratch_bytes=mid)
            hi = mid
        except RuntimeError as e:
            assert "invalidArg" in str(e) or "INVALID" in str(e).upper(), e
            lo = mid + 1
    return lo


def test_slices(S, oc):
    """a scratch for one block, for a few blocks and for the whole batch gives the same frames; dependent frames with block
    checksums straddle the slice boundaries"""
    text = dict(K.frame_inputs())["text"]
    rng = random.Random(9)
    units = [text[:n] for n in (0, 1000, 1024, 1025, 5000, 17000)] + [H.random_bytes(rng, 3000), text[7:40000]]
    for ind in (False, True):
        opts = dict(independentBlocks=ind, blockChecksums=True, contentChecksum=True, contentSize=True, blockSize=1024)
        b, st, ln, whole = _frames(units, opts)
        _check(oc, units, st, ln, whole, opts)
        full = b.d_scratch.numel()
        nblk = sum(-(-len(u) // 1024) for u in units)
        one = _min_scratch(units, opts)
        need = (full - one) // (nblk - 1)
        assert one + (nblk - 1) * need == full
        for scr in (one, one + 4 * need, one + 4 * need + need // 2, full):
            _, st2, ln2, outs2 = _frames(units, opts, scratch_bytes=scr)
            assert (st2 == st).all() and (ln2 == ln).all() and outs2 == whole, scr


def test_max_blocks(S, oc):
    """the block table fills in unit order: a table too small gives the later units SWC_ERR_UNSUPPORTED and nothing written,
    the earlier ones their frames; max_blocks == 0 (the library counts) gives what the exact count gives"""
    text = dict(K.frame_inputs())["text"]
    units = [text[:3000], text[:10000], b"", text[5:9000], text[:1], text[:4000]]       # 3, 10, 0, 9, 1, 4 blocks of 1 KiB
    opts = dict(independentBlocks=False, blockChecksums=True, contentChecksum=True, contentSize=False, blockSize=1024)
    b, st, ln, outs = _frames(units, opts, max_blocks=None)
    _check(oc, units, st, ln, outs, opts)
    _, st1, ln1, outs1 = _frames(units, opts, max_blocks=27)
    assert (st1 == st).all() and (ln1 == ln).all() and outs1 == outs
    from swcompression_b200.batch import Batch
    t = Batch.from_units("lz4_frame_compress", units, np.array([_bound(len(u), opts) for u in units], dtype=np.uint64),
                         max_blocks=20, block_size=1024, frame_flags={k: v for k, v in opts.items() if k != "blockSize"})
    t.d_out.fill_(H.SENTINEL)
    t.run()
    st2, ln2, _ = t.results()
    assert list(st2) == [OK, OK, OK, UNSUPPORTED, UNSUPPORTED, UNSUPPORTED]
    host = t.d_out.cpu().numpy()
    for i in range(6):
        o = int(t.h_out_off[i])
        if i < 3:
            assert bytes(host[o:o + int(ln2[i])]) == outs[i] and ln2[i] == ln[i]
        else:
            assert ln2[i] == 0 and (host[o:o + int(t.h_out_cap[i])] == H.SENTINEL).all(), i


def test_graph_capture(S, oc):
    """with caller scratch and max_blocks the call reads nothing back: captured into a CUDA graph, a replay on new bytes of
    the same lengths gives the new bytes' frames, and the launch count does not depend on the data"""
    import torch
    from swcompression_b200 import _lib
    from swcompression_b200.batch import Batch, pack_units
    rng = random.Random(13)
    text = dict(K.frame_inputs())["text"]
    lens = [0, 1, 700, 4096, 4097, 20000, 65536, 70001]
    first = [text[:n] for n in lens]
    second = [H.random_bytes(rng, n) if k % 2 else text[::-1][:n] for k, n in enumerate(lens)]
    opts = dict(independentBlocks=False, blockChecksums=True, contentChecksum=True, contentSize=True, blockSize=4096)
    flags = {k: v for k, v in opts.items() if k != "blockSize"}
    caps = np.array([_bound(n, opts) for n in lens], dtype=np.uint64)
    b = Batch.from_units("lz4_frame_compress", first, caps, block_size=4096, frame_flags=flags, max_blocks=64)
    L = _lib.lib()
    n0 = L.swc_kernel_launches()
    b.run()
    st0, ln0, _ = b.results()
    eager = L.swc_kernel_launches() - n0
    _check(oc, first, st0, ln0, b.outputs(), opts)
    b.d_status.fill_(-1); b.d_out_len.zero_(); b.d_out.zero_()
    torch.cuda.synchronize()
    s = torch.cuda.Stream()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.stream(s):
        with torch.cuda.graph(g, stream=s):
            b.run()
    torch.cuda.synchronize()
    assert (b.d_status.cpu().numpy() == -1).all()
    buf, _, _ = pack_units(second)
    b.d_in.copy_(torch.from_numpy(buf).cuda())
    g.replay()
    st1, ln1, _ = b.results()
    _check(oc, second, st1, ln1, b.outputs(), opts)
    n1 = L.swc_kernel_launches()
    b.run()
    b.results()
    assert L.swc_kernel_launches() - n1 == eager


def test_benched_shape(S, oc):
    """tiled copies of the benchmark's 16 MiB frames of 64 KiB blocks: every copy equals the first on the device, the first
    the oracle"""
    import torch
    from swcompression_b200.batch import Batch
    rng = random.Random(4)
    distinct = []
    for i in range(64):
        r = i % 10
        distinct.append(bytes(65536) if r == 8 else H.random_bytes(rng, 65536) if r == 9 else H.textlike(65536, 500 + i))
    frame = b"".join(distinct) * 4
    tile = 16
    buf = np.frombuffer(frame * tile + bytes(64), dtype=np.uint8)
    offs = np.arange(tile, dtype=np.uint64) * np.uint64(len(frame))
    opts = dict(K.TRICKY_OPTS, independentBlocks=True, blockSize=65536)
    cap = _bound(len(frame), opts)
    b = Batch("lz4_frame_compress", buf, offs, np.full(tile, len(frame), dtype=np.uint64), cap, block_size=65536,
              frame_flags={k: v for k, v in opts.items() if k != "blockSize"}, max_blocks=tile * 256)
    b.run()
    st, ln, _ = b.results()
    assert (st == OK).all() and (ln == ln[0]).all()
    stride = (cap + 15) // 16 * 16
    out = b.d_out[: tile * stride].view(tile, stride)[:, : int(ln[0])]
    assert bool((out == out[0:1]).all())
    assert bytes(out[0].cpu().numpy()) == oc.lz4_compress(frame, **opts)[1]
    del out, b
    torch.cuda.empty_cache()
