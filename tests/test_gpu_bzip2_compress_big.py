"""The CUDA BZip2 compressor on the full-size cases of bzip2c_big_cases.py (15-17 doubling rounds of sort_kernel, keys
spanning more than the block, whole-block ties, RLE1 output at rle_cap, 256 used bytes and 6 tables, a unit of blocks with
very different round counts), byte for byte against the CPU restatement of BZip2+Compress.swift, in plain and hostile
batches, with capacities exactly out_len and one byte short, through the single call, and back through the engine's
decoder and Python's bz2."""
import bz2
import random

import numpy as np
import pytest

import bzip2c_big_cases as K
import compress_batch as CB
import helpers as H

pytestmark = pytest.mark.gpu

LEVELS = sorted({k for _, _, k in K.cases()})


@pytest.fixture(scope="module")
def oc():
    import swco_bzip2c
    swco_bzip2c.lib()
    return swco_bzip2c


@pytest.fixture(scope="module")
def gpu():
    import torch
    assert torch.cuda.is_available()
    import swcompression_b200 as S
    return S


_EXP = {}


def expected(oc, name):
    if name not in _EXP:
        data, k = K.by_name()[name]
        st, out, _ = oc.bzip2_compress(data, k)
        assert st == 0
        _EXP[name] = out
    return _EXP[name]


def level(k):
    return [(name, data) for name, data, kk in K.cases() if kk == k]


@pytest.mark.parametrize("k", LEVELS)
def test_level_batch(gpu, oc, k):
    """each level's cases as one batch, then the streams through the engine's BZip2 decoder and bz2"""
    from swcompression_b200.batch import Batch
    items = level(k)
    units = [d for _, d in items]
    b = Batch.from_units("bzip2_compress", units, [gpu.BZip2.max_compressed_size(len(u), k) for u in units], block_size=k)
    b.run()
    st, ln, _ = b.results()
    outs = b.outputs()
    for (name, u), s, l, o in zip(items, st, ln, outs):
        exp = expected(oc, name)
        assert s == 0 and l == len(exp) and o == exp, name
    d = Batch.from_units("bzip2", outs, [max(len(u), 16) for u in units])
    d.run()
    dst, _, _ = d.results()
    assert (dst == 0).all() and d.outputs() == units
    for o, u in zip(outs, units):
        assert bz2.decompress(o) == u


@pytest.mark.parametrize("k", LEVELS)
def test_level_fenced(gpu, oc, k):
    """compress_batch.fenced's hostile layout.  runs4_k9 goes first, where its capacity is exact: its RLE1 output fills
    its block scratch to rle_cap, directly in front of every other unit's blocks"""
    items = sorted(level(k), key=lambda it: it[0] != "runs4_k9")
    CB.fenced("bzip2_compress", k, [d for _, d in items], exp=[expected(oc, name) for name, _ in items])


@pytest.mark.parametrize("k", LEVELS)
def test_twice_exact_and_one_short(gpu, oc, k):
    """every case three times in one batch, packed hostile: in order and in reverse with capacity exactly out_len (equal
    outputs at different offsets, next to different neighbours), then in order with out_len - 1, which is
    SWC_ERR_OUTPUT_OVERFLOW with the exact out_len and no byte written; output regions one byte apart"""
    from swcompression_b200.batch import compress_scratch_bytes
    items = level(k)
    exp = [expected(oc, name) for name, _ in items]
    units = [d for _, d in items] + [d for _, d in items[::-1]] + [d for _, d in items]
    want = exp + exp[::-1] + exp
    caps = np.array([len(e) for e in exp + exp[::-1]] + [len(e) - 1 for e in exp], dtype=np.uint64)
    in_buf, in_off, in_len = H.pack_hostile(units, random.Random(k))
    out_off = np.zeros(len(units), dtype=np.uint64)
    pos = H.GUARD
    for j, c in enumerate(caps.tolist()):
        out_off[j] = pos
        pos += c + 1
    total = pos + H.GUARD
    rc, st, ln, out, _ = CB.run_batch("bzip2_compress", k, in_buf, in_off, in_len, out_off, caps, total,
                                      compress_scratch_bytes("bzip2_compress", in_len, block_size=k))
    assert rc == 0
    assert ln.tolist() == [len(e) for e in want]
    written = np.zeros(total, dtype=bool)
    for j, e in enumerate(want):
        o = int(out_off[j])
        if j < 2 * len(items):
            assert st[j] == 0 and bytes(out[o:o + len(e)]) == e, (j, items[j % len(items)][0])
            written[o:o + len(e)] = True
        else:
            assert st[j] == CB.OVERFLOW, j
    assert (out[~written] == H.SENTINEL).all()


@pytest.mark.parametrize("name", K.MANY_ROUNDS + K.EXPANSION)
def test_single_call(gpu, oc, name):
    data, k = K.by_name()[name]
    got = gpu.BZip2.compress(data, gpu.BZip2.BlockSize(k))
    assert got == expected(oc, name)
    assert bz2.decompress(got) == data
