"""The link-builder and emit-chunk catalogue (compress_link_cases.py) through the CUDA compressors,
swc_deflate_compress_batch and swc_lz4_block_compress_batch (LZ4 also through frames), byte for byte against the CPU
restatements of the reference: in one slice on a caller scratch, in slices of a small scratch, and packed hostile into
fenced output regions; then back through the engine's own decoders.  The catalogue's units sit between runs of 0-, 1-
and 2-byte units, which have no link tiles (and, beyond 4 GiB, no emit chunks either)."""
import ctypes as C
import random

import numpy as np
import pytest

import compress_batch as CB
import compress_link_cases as K
import helpers as H

pytestmark = pytest.mark.gpu

UNSUPPORTED = 6
TINY_RUNS = ([], [b""], [b"", b"a", b"ab"], [b"ab", b"ab"], [b"a"], [b"", b""])


@pytest.fixture(scope="module")
def gpu():
    import torch
    assert torch.cuda.is_available()
    import swcompression_b200 as S
    return S


def with_tiny_runs(units):
    """`units` with runs of zero-tile units in front of, between and behind them"""
    out = []
    for k, u in enumerate(units):
        out += TINY_RUNS[k % len(TINY_RUNS)] + [u]
    return out + [b"", b"a", b"ab"]


def launches():
    from swcompression_b200 import _lib
    return _lib.lib().swc_kernel_launches()


def run(codec, d_in, in_off, in_len, out_off, out_cap, total, scratch, dict_off=None, dict_len=None):
    """one batch call on a device input -> (return code, status, out_len, output buffer, kernel launches)"""
    import torch
    from swcompression_b200 import _lib
    dev = d_in.device
    t = lambda a: torch.from_numpy(np.ascontiguousarray(a, dtype=np.uint64).view(np.int64)).to(dev)
    n = len(in_off)
    d_out = torch.full((total,), H.SENTINEL, dtype=torch.uint8, device=dev)
    d_len, d_st = torch.zeros(n, dtype=torch.int64, device=dev), torch.full((n,), -1, dtype=torch.int32, device=dev)
    scr = torch.empty(scratch, dtype=torch.uint8, device=dev)
    i_off, i_len, o_off, o_cap = t(in_off), t(in_len), t(out_off), t(out_cap)
    p = lambda x: None if x is None else C.c_void_p(x.data_ptr())
    s = C.c_void_p(torch.cuda.current_stream(dev).cuda_stream)
    L = _lib.lib()
    before = launches()
    if codec == "deflate_compress":
        rc = L.swc_deflate_compress_batch(p(d_in), p(i_off), p(i_len), p(d_out), p(o_off), p(o_cap), p(d_len), p(d_st), n,
                                          p(scr), scratch, s)
    else:
        dofs = None if dict_off is None else t(dict_off)
        dlns = None if dict_len is None else t(dict_len)
        rc = L.swc_lz4_block_compress_batch(p(d_in), p(i_off), p(i_len), p(dofs), p(dlns), p(d_out), p(o_off), p(o_cap),
                                            p(d_len), p(d_st), n, p(scr), scratch, s)
    n_launch = launches() - before
    torch.cuda.synchronize()
    return rc, d_st.cpu().numpy(), d_len.cpu().numpy(), d_out.cpu().numpy(), n_launch


def check_fenced(exp, st, ln, out, out_off, out_cap):
    """`exp`: each unit's stream, or a status for a unit that must fail with out_len 0 and write nothing"""
    written = np.zeros(len(out), dtype=bool)
    for j, e in enumerate(exp):
        o = int(out_off[j])
        if isinstance(e, int):
            assert st[j] == e and ln[j] == 0, j
            continue
        assert ln[j] == len(e), j
        if out_cap[j] < len(e):
            assert st[j] == CB.OVERFLOW, j
        else:
            assert st[j] == 0 and bytes(out[o:o + len(e)]) == e, j
            written[o:o + len(e)] = True
    assert (out[~written] == H.SENTINEL).all()


# ---- Deflate -----------------------------------------------------------------------------------------------------------

def deflate_units():
    return with_tiny_runs([d for _, d, _ in K.deflate_cases()])


def test_deflate_cases_one_slice_and_round_trip(gpu):
    """the plain layout on a caller scratch that runs it in one slice, then back through the batch decoder"""
    import swco_deflatec
    from swcompression_b200.batch import Batch
    units = deflate_units()
    exp = [swco_deflatec.deflate_compress(u)[1] for u in units]
    b = Batch.from_units("deflate_compress", units, [(9 * len(u) + 17) // 8 for u in units])
    before = launches()
    b.run()
    assert launches() - before == CB.LAUNCHES["deflate_compress"]
    st, ln, _ = b.results()
    outs = b.outputs()
    for k, (o, e) in enumerate(zip(outs, exp)):
        assert st[k] == 0 and o == e, k
    d = Batch.from_units("deflate", outs, [max(len(u), 16) for u in units])
    d.run()
    dst, _, _ = d.results()
    assert (dst == 0).all() and d.outputs() == units


def test_deflate_cases_fenced_in_one_slice_and_in_slices(gpu):
    """hostile packing and fenced outputs, once in one slice and once on a scratch that holds only the largest unit"""
    import swco_deflatec
    from swcompression_b200.batch import compress_scratch_bytes
    units = deflate_units()
    exp = [swco_deflatec.deflate_compress(u)[1] for u in units]
    a = CB.fenced("deflate_compress", 1, units, exp=exp)
    assert a[3] == CB.LAUNCHES["deflate_compress"]
    small = compress_scratch_bytes("deflate_compress", [max(len(u) for u in units)])
    b = CB.fenced("deflate_compress", 1, units, scratch=small, exp=exp)
    assert b[3] > a[3]
    for x, y in zip(a[:3], b[:3]):
        assert (x == y).all()


def test_deflate_unit_of_4_gib_is_unsupported(gpu):
    """a real 2^32-byte unit between catalogue units and tiny ones: SWC_ERR_UNSUPPORTED, out_len 0, nothing written, and
    every other unit exact (the unit has neither link tiles nor emit chunks)"""
    import torch
    import swco_deflatec
    from swcompression_b200.batch import compress_scratch_bytes
    names = ("halo_x0_d32768", "chunk_boundaries", "phase_7")
    cases = {c[0]: c[1] for c in K.deflate_cases()}
    small = [b"", b"a", cases[names[0]], b"ab", b""] + [cases[names[1]], b"a", b"ab", cases[names[2]], b""]
    at = 5                                                        # the 4 GiB unit goes in front of small[at]
    exp = [swco_deflatec.deflate_compress(u)[1] for u in small]
    exp.insert(at, UNSUPPORTED)
    buf, offs, lens = H.pack_hostile(small, random.Random(9))
    big_off = (len(buf) + 15) // 16 * 16
    dev = torch.device("cuda:0")
    d_in = torch.zeros(big_off + K.MAX_UNIT + 64, dtype=torch.uint8, device=dev)
    d_in[:len(buf)] = torch.from_numpy(buf).to(dev)
    in_off = np.insert(offs, at, np.uint64(big_off))
    in_len = np.insert(lens, at, np.uint64(K.MAX_UNIT))
    out_off, out_cap, total = H.fenced_layout([64 if isinstance(e, int) else len(e) for e in exp], align=16)
    scratch = compress_scratch_bytes("deflate_compress", np.insert(lens, at, np.uint64(0)))
    try:
        rc, st, ln, out, n_launch = run("deflate_compress", d_in, in_off, in_len, out_off, out_cap, total, scratch)
        assert rc == 0 and n_launch == CB.LAUNCHES["deflate_compress"]
        check_fenced(exp, st, ln, out, out_off, out_cap)
    finally:
        del d_in
        torch.cuda.empty_cache()


# ---- LZ4 ---------------------------------------------------------------------------------------------------------------

def test_lz4_cases_without_dictionary(gpu):
    """the block cases with no dictionary: plain in one slice and back through the block decoder, fenced in one slice
    and in slices"""
    import swco_lz4c
    from swcompression_b200.batch import Batch, compress_scratch_bytes
    units = with_tiny_runs([blk for _, blk, d, _ in K.lz4_cases() if not d])
    exp = [swco_lz4c.lz4_block_compress(u)[1] for u in units]
    b = Batch.from_units("lz4_block_compress", units, [len(u) + len(u) // 255 + 16 for u in units])
    before = launches()
    b.run()
    assert launches() - before == CB.LAUNCHES["lz4_block_compress"]
    st, _, _ = b.results()
    outs = b.outputs()
    assert (st == 0).all() and outs == exp
    d = Batch.from_units("lz4_block", outs, [max(len(u), 16) for u in units])
    d.run()
    dst, _, _ = d.results()
    assert (dst == 0).all() and d.outputs() == units
    a = CB.fenced("lz4_block_compress", 1, units, exp=exp)
    assert a[3] == CB.LAUNCHES["lz4_block_compress"]
    small = compress_scratch_bytes("lz4_block_compress", [max(len(u) for u in units)])
    s = CB.fenced("lz4_block_compress", 1, units, scratch=small, exp=exp)
    assert s[3] > a[3]
    for x, y in zip(a[:3], s[:3]):
        assert (x == y).all()


def pack_windows(pairs, rng):
    """(block, dictionary) pairs -> input buffer with each dictionary directly in front of its block and junk of every
    length 1-16 in front of each window -> (buffer, in_off, in_len, dict_off, dict_len)"""
    buf = bytearray(b"\xFF" * 16)
    in_off, dict_off = [], []
    for k, (blk, d) in enumerate(pairs):
        buf += bytes(rng.randrange(1, 256) for _ in range(1 + k % 16))
        dict_off.append(len(buf))
        buf += d
        in_off.append(len(buf))
        buf += blk
    buf += b"\xFF" * H.GUARD
    return (np.frombuffer(bytes(buf), dtype=np.uint8).copy(), np.array(in_off, dtype=np.uint64),
            np.array([len(b) for b, _ in pairs], dtype=np.uint64), np.array(dict_off, dtype=np.uint64),
            np.array([len(d) for _, d in pairs], dtype=np.uint64))


def test_lz4_dictionary_windows_fenced(gpu):
    """the seam cases (and the others with no dictionary) as windows into one input, fenced, in one slice and in
    slices of a scratch that holds only the largest window"""
    import torch
    import swco_lz4c
    from swcompression_b200.batch import compress_scratch_bytes
    pairs = []
    for k, (_, blk, d, _) in enumerate(K.lz4_cases()):
        pairs += [(u, b"") for u in TINY_RUNS[k % len(TINY_RUNS)]] + [(blk, d)]
    exp = [swco_lz4c.lz4_block_compress(b, d)[1] for b, d in pairs]
    buf, in_off, in_len, d_off, d_len = pack_windows(pairs, random.Random(13))
    d_in = torch.from_numpy(buf).to("cuda:0")
    out_off, out_cap, total = H.fenced_layout([len(e) for e in exp], align=1)
    full = compress_scratch_bytes("lz4_block_compress", in_len, dict_len=d_len)
    k = int(np.argmax(in_len + np.minimum(d_len, np.uint64(K.MAX_DICT))))
    small = compress_scratch_bytes("lz4_block_compress", [in_len[k]], dict_len=[d_len[k]])
    results = []
    for scratch in (full, small):
        rc, st, ln, out, n_launch = run("lz4_block_compress", d_in, in_off, in_len, out_off, out_cap, total, scratch,
                                        d_off, d_len)
        assert rc == 0
        check_fenced(exp, st, ln, out, out_off, out_cap)
        results.append((st, ln, out, n_launch))
    assert results[0][3] == CB.LAUNCHES["lz4_block_compress"] < results[1][3]


@pytest.mark.parametrize("name", [c[0] for c in K.lz4_cases()])
def test_lz4_cases_in_frames(gpu, name):
    """each case as a one-block frame (its dictionary as the frame's), against the restatement and back"""
    import swco_lz4c
    _, blk, d, _ = {c[0]: c for c in K.lz4_cases()}[name]
    opts = dict(independentBlocks=True, blockChecksums=True, contentChecksum=True, contentSize=True)
    if d:
        opts["dictionary"] = d
    st, exp, _ = swco_lz4c.lz4_compress(blk, **opts)
    assert st == 0
    got = gpu.LZ4.compress(blk, **opts)
    assert got == exp
    assert gpu.LZ4.decompress(got, dictionary=d or None) == blk


def test_lz4_blocks_of_4_mib_and_one_more(gpu):
    """a block of exactly MAX_BLOCK bytes compresses; one byte more is SWC_ERR_UNSUPPORTED with out_len 0 and nothing
    written, in the same batch"""
    import swco_lz4c
    text = H.textlike(K.MAX_BLOCK + 1, 31)
    case = K.lz4_cases()[0][1]
    units = [b"a", text[:K.MAX_BLOCK], b"", text[::-1], case]
    exp = [swco_lz4c.lz4_block_compress(u)[1] for u in units]
    exp[3] = UNSUPPORTED
    buf, in_off, in_len = H.pack_hostile(units, random.Random(3))
    import torch
    from swcompression_b200.batch import compress_scratch_bytes
    out_off, out_cap, total = H.fenced_layout([64 if isinstance(e, int) else len(e) for e in exp], align=1)
    rc, st, ln, out, n_launch = run("lz4_block_compress", torch.from_numpy(buf).to("cuda:0"), in_off, in_len, out_off,
                                    out_cap, total, compress_scratch_bytes("lz4_block_compress", in_len))
    assert rc == 0 and n_launch == CB.LAUNCHES["lz4_block_compress"]
    check_fenced(exp, st, ln, out, out_off, out_cap)
