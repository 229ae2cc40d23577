"""The batch contract the three compressors share (swc_lz4_block_compress_batch, swc_deflate_compress_batch,
swc_bzip2_compress_batch in include/swcgpu.h), checked against each codec's CPU restatement of the reference.  Each
codec's test file runs these checks for its codec:

- inputs packed with no friendly bytes around them (helpers.pack_hostile);
- output regions with exact capacities, 1-15 bytes short and 1-15 bytes long, at every start residue the codec allows;
- out_len exact also on overflow, an overflowing unit writes nothing, and no byte changes outside what the units that
  succeed produce;
- the slice policy: a scratch of *_scratch_bytes(n, ...) runs the batch in one slice, a smaller one that holds the
  largest unit runs it in several with identical results, and one below the largest unit's need is SWC_ERR_INVALID_ARG."""
import ctypes as C
import functools
import random

import numpy as np

import deflatec_cases as DK
import helpers as H
import lz4c_cases as LK

ALIGN = {"lz4_block_compress": 1, "deflate_compress": 16, "bzip2_compress": 1}       # output starts each contract allows
LAUNCHES = {"lz4_block_compress": 3, "deflate_compress": 4, "bzip2_compress": 9}     # kernel launches of one slice
OVERFLOW, INVALID_ARG = 1, 4


def expected(codec, k, units):
    if codec == "lz4_block_compress":
        import swco_lz4c
        return [swco_lz4c.lz4_block_compress(u)[1] for u in units]
    if codec == "deflate_compress":
        import swco_deflatec
        return [swco_deflatec.deflate_compress(u)[1] for u in units]
    import swco_bzip2c
    return [swco_bzip2c.bzip2_compress(u, k)[1] for u in units]


@functools.lru_cache(maxsize=None)
def mixed_units():
    """the units every codec's batch test ran before they shared this file, together: short strings, zeros, a two-block
    BZip2 unit, a Deflate unit one byte past a link tile, and the random and text slices each drew from
    random.Random(17)"""
    text = H.textlike(200000, 21)
    lz4_text = dict(LK.frame_inputs())["text"]
    units = [b"", b"a", b"abcabcabcabc", b"abcdabcdabcdabcd", text[:1000], bytes(5000), text[3:70000], text[3:90000],
             text[:DK.TILE + 1], bytes(range(200, 256))]
    for n_rand, src, n_slices in ((10, text, 40), (8, text, 30), (10, lz4_text, 30)):     # Deflate's, BZip2's, LZ4's
        rng = random.Random(17)
        units += [bytes(rng.getrandbits(8) for _ in range(rng.randint(0, 3000))) for _ in range(n_rand)]
        units += [src[rng.randint(0, 10000):][:rng.randint(1, 9000)] for _ in range(n_slices)]
    return tuple(units)


def run_batch(codec, k, in_buf, in_off, in_len, out_off, out_cap, out_total, scratch):
    """-> (return code, status, out_len, output buffer, kernel launches)"""
    import torch
    from swcompression_b200 import _lib
    dev = torch.device("cuda:0")
    t = lambda a: torch.from_numpy(np.ascontiguousarray(a, dtype=np.uint64).view(np.int64)).to(dev)
    n = len(in_off)
    d_in = torch.from_numpy(in_buf).to(dev)
    d_out = torch.full((out_total,), H.SENTINEL, dtype=torch.uint8, device=dev)
    d_len, d_st = torch.zeros(n, dtype=torch.int64, device=dev), torch.full((n,), -1, dtype=torch.int32, device=dev)
    scr = torch.empty(scratch, dtype=torch.uint8, device=dev)
    i_off, i_len, o_off, o_cap = t(in_off), t(in_len), t(out_off), t(out_cap)
    p = lambda x: C.c_void_p(x.data_ptr())
    s = C.c_void_p(torch.cuda.current_stream(dev).cuda_stream)
    L = _lib.lib()
    before = L.swc_kernel_launches()
    if codec == "lz4_block_compress":
        rc = L.swc_lz4_block_compress_batch(p(d_in), p(i_off), p(i_len), None, None, p(d_out), p(o_off), p(o_cap), p(d_len),
                                            p(d_st), n, p(scr), scratch, s)
    elif codec == "deflate_compress":
        rc = L.swc_deflate_compress_batch(p(d_in), p(i_off), p(i_len), p(d_out), p(o_off), p(o_cap), p(d_len), p(d_st), n,
                                          p(scr), scratch, s)
    else:
        rc = L.swc_bzip2_compress_batch(p(d_in), p(i_off), p(i_len), k, p(d_out), p(o_off), p(o_cap), p(d_len), p(d_st), n,
                                        p(scr), scratch, s)
    launches = L.swc_kernel_launches() - before
    torch.cuda.synchronize()
    return rc, d_st.cpu().numpy(), d_len.cpu().numpy(), d_out.cpu().numpy(), launches


def fenced(codec, k, units, scratch=None, exp=None):
    """runs `units` packed hostile into fenced output regions and checks every result and the fence; `exp` are the
    expected streams when the caller has them already -> (status, out_len, output buffer, kernel launches)"""
    from swcompression_b200.batch import compress_scratch_bytes
    exp = expected(codec, k, units) if exp is None else exp
    in_buf, in_off, in_len = H.pack_hostile(units, random.Random(5))
    out_off, out_cap, total = H.fenced_layout([len(e) for e in exp], align=ALIGN[codec])
    if scratch is None:
        scratch = compress_scratch_bytes(codec, in_len, block_size=k)
    rc, st, ln, out, launches = run_batch(codec, k, in_buf, in_off, in_len, out_off, out_cap, total, scratch)
    assert rc == 0
    written = np.zeros(total, dtype=bool)
    for j, e in enumerate(exp):
        o = int(out_off[j])
        assert ln[j] == len(e), j
        if out_cap[j] < len(e):
            assert st[j] == OVERFLOW, j
        else:
            assert st[j] == 0 and bytes(out[o:o + len(e)]) == e, j
            written[o:o + len(e)] = True
    assert (out[~written] == H.SENTINEL).all()
    return st, ln, out, launches


def one_slice(codec, k=1):
    """*_scratch_bytes(n, ...) runs the mixed batch in one slice"""
    assert fenced(codec, k, mixed_units())[3] == LAUNCHES[codec]


def in_slices(codec, k=1):
    """a scratch that holds the largest unit but not the batch runs it in slices: the results must not change"""
    from swcompression_b200.batch import compress_scratch_bytes
    units = mixed_units()
    full = compress_scratch_bytes(codec, [len(u) for u in units], block_size=k)
    small = compress_scratch_bytes(codec, [max(len(u) for u in units)], block_size=k)
    assert small < full
    a = fenced(codec, k, units)
    b = fenced(codec, k, units, scratch=small)
    assert b[3] > a[3] == LAUNCHES[codec]
    for x, y in zip(a[:3], b[:3]):
        assert (x == y).all()


def tiny_units_one_slice(codec, k=1):
    """*_scratch_bytes is enough for one slice also for batches of tiny units, around one unit of a full BZip2 block"""
    rng = random.Random(23)
    for units in ([bytes(rng.getrandbits(8) for _ in range(rng.randint(0, 84))) for _ in range(300)],
                  [b"x"] * 50 + [H.textlike(80001, 3)] + [bytes(200)] * 50):
        assert fenced(codec, k, units)[3] == LAUNCHES[codec]


def below_largest_unit_is_invalid(codec, k=1):
    """a caller scratch smaller than what the largest unit needs alone is SWC_ERR_INVALID_ARG"""
    from swcompression_b200.batch import compress_scratch_bytes
    units = mixed_units()
    in_buf, in_off, in_len = H.pack_hostile(units, random.Random(5))
    out_off, out_cap, total = H.fenced_layout([2 * len(u) + 1024 for u in units], align=ALIGN[codec])
    # a quarter of the one-unit bound is below the need of the 89 997-byte unit for every codec
    scratch = compress_scratch_bytes(codec, [int(in_len.max())], block_size=k) // 4
    assert run_batch(codec, k, in_buf, in_off, in_len, out_off, out_cap, total, scratch)[0] == INVALID_ARG
