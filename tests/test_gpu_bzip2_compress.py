"""The CUDA BZip2 compressor (bzip2_compress.cu through swc_bzip2_compress_batch and the single call) byte for byte
against the CPU restatement of BZip2+Compress.swift, and back through the engine's own decoder and Python's bz2."""
import bz2
import ctypes as C
import random

import numpy as np
import pytest

import bzip2c_cases as K
import compress_batch as CB
import helpers as H

pytestmark = pytest.mark.gpu


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


def test_catalogue_batch(gpu, oc):
    from swcompression_b200.batch import Batch
    by_level = {}
    for name, data, k in K.cases():
        by_level.setdefault(k, []).append((name, data))
    by_level.setdefault(1, []).extend((a, H.answer(a)) for a in ("test1", "test5", "test6"))
    for k, items in sorted(by_level.items()):
        units = [d for _, d in items]
        b = Batch.from_units("bzip2_compress", units, [gpu.BZip2.max_compressed_size(len(u), k) for u in units], block_size=k)
        b.run()
        st, ln, _ = b.results()
        outs = b.outputs()
        for (name, u), s, l, o in zip(items, st, ln, outs):
            ost, exp, _ = oc.bzip2_compress(u, k)
            assert s == ost == 0 and l == len(exp) and o == exp, name
        d = Batch.from_units("bzip2", outs, [max(len(u), 16) for u in units])
        d.run()
        dst, _, _ = d.results()
        assert (dst == 0).all() and d.outputs() == units


@pytest.mark.parametrize("k", [1, 5, 9])
def test_single_calls(gpu, oc, k):
    S = gpu
    rng = np.random.default_rng(k)
    for data in [H.textlike(24 << 20, 5 + k), bytes(64 << 20), rng.bytes(4 << 20)]:
        got = S.BZip2.compress(data, S.BZip2.BlockSize(k))
        assert got == oc.bzip2_compress(data, k)[1], len(data)
        assert bz2.decompress(got) == data
        assert len(got) <= S.BZip2.max_compressed_size(len(data), k)


def test_default_block_size_and_invalid(gpu):
    S = gpu
    assert S.BZip2.compress(b"hello hello") == S.BZip2.compress(b"hello hello", S.BZip2.BlockSize.one)
    from swcompression_b200 import _lib
    L = _lib.lib()
    out, ln = C.c_void_p(), C.c_size_t(0)
    for bad in (0, 10, -1):
        assert L.swc_bzip2_compress(b"abc", 3, bad, C.byref(out), C.byref(ln)) == 4   # SWC_ERR_INVALID_ARG
        assert L.swc_bzip2_compress_batch(None, None, None, bad, None, None, None, None, None, 1, None, 0, None) == 4


# ---- the batch layout and slice contract it shares with LZ4 and Deflate (compress_batch.py) ----------------------------

def test_batch_fenced(gpu):
    CB.one_slice("bzip2_compress", 1)


def test_batch_fenced_in_slices(gpu):
    """the two-block unit (about 3.5 MiB of scratch) fits a slice alone, the batch does not"""
    CB.in_slices("bzip2_compress", 1)


def test_scratch_bytes_run_one_slice(gpu):
    CB.tiny_units_one_slice("bzip2_compress", 1)


@pytest.mark.parametrize("k", [1, 5])
def test_scratch_below_largest_unit_is_invalid(gpu, k):
    CB.below_largest_unit_is_invalid("bzip2_compress", k)


def test_batch_contract_at_block_size_5(gpu):
    CB.in_slices("bzip2_compress", 5)
    CB.tiny_units_one_slice("bzip2_compress", 5)


def test_benched_shape_tiled(gpu, oc):
    """80 000-byte units at .one in the benchmark's mix, tiled: equal outputs across tiles, the oracle on distinct units"""
    from swcompression_b200.batch import Batch
    rng = random.Random(4)
    U = 80000
    distinct = []
    for i in range(40):
        r = i % 10
        distinct.append(bytes(U) if r == 8 else bytes(rng.getrandbits(8) for _ in range(U)) if r == 9
                        else H.textlike(U, 700 + i))
    tile = 50
    buf = np.frombuffer(b"".join(distinct) * tile + bytes(64), dtype=np.uint8)
    offs = np.arange(40 * tile, dtype=np.uint64) * np.uint64(U)
    cap = gpu.BZip2.max_compressed_size(U, 1)
    b = Batch("bzip2_compress", buf, offs, np.full(40 * tile, U, dtype=np.uint64), cap, block_size=1)
    b.run()
    st, ln, _ = b.results()
    assert (st == 0).all()
    assert (ln.reshape(tile, 40) == ln[:40][None, :]).all()
    outs = b.outputs()
    for j in range(40 * tile):
        assert outs[j] == outs[j % 40], j
    for j, u in enumerate(distinct):
        assert outs[j] == oc.bzip2_compress(u, 1)[1], j
