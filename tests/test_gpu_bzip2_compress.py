"""The CUDA BZip2 compressor (bzip2_compress.cu through swc_bzip2_compress_batch and the single call) byte for byte
against the CPU restatement of BZip2+Compress.swift, and back through the engine's own decoder and Python's bz2."""
import bz2
import ctypes as C
import random

import numpy as np
import pytest

import bzip2c_cases as K
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


def run_batch(units, in_offs, in_buf, out_off, out_cap, out_total, k, scratch=None, fill=0xA5):
    import torch
    from swcompression_b200 import _lib
    dev = torch.device("cuda:0")
    t = lambda a: torch.from_numpy(np.asarray(a, dtype=np.uint64).view(np.int64)).to(dev)
    n = len(units)
    d_in = torch.from_numpy(in_buf).to(dev)
    d_out = torch.full((out_total,), fill, dtype=torch.uint8, device=dev)
    lens = np.array([len(u) for u in units], dtype=np.uint64)
    d_len, d_st = torch.zeros(n, dtype=torch.int64, device=dev), torch.full((n,), -1, dtype=torch.int32, device=dev)
    L = _lib.lib()
    nb = L.swc_bzip2_compress_batch_scratch_bytes(n, int(lens.sum()), k) if scratch is None else scratch
    scr = torch.empty(nb, dtype=torch.uint8, device=dev)
    keep = [t(in_offs), t(lens), t(out_off), t(out_cap)]
    p = lambda x: C.c_void_p(x.data_ptr())
    st = L.swc_bzip2_compress_batch(p(d_in), p(keep[0]), p(keep[1]), k, p(d_out), p(keep[2]), p(keep[3]), p(d_len), p(d_st),
                                    n, p(scr), scr.numel(), C.c_void_p(torch.cuda.current_stream(dev).cuda_stream))
    assert st == 0
    torch.cuda.synchronize()
    return d_st.cpu().numpy(), d_len.cpu().numpy(), d_out.cpu().numpy()


def fenced(oc, scratch=None, k=1):
    """unaligned back-to-back inputs; output regions at any alignment with capacities exact, 1-15 short and 1-15 long"""
    rng = random.Random(17)
    text = H.textlike(200000, 21)
    units = [b"", b"a", b"abcabcabcabc", text[:1000], bytes(5000), text[3:90000], bytes(range(200, 256))]
    units += [bytes(rng.getrandbits(8) for _ in range(rng.randint(0, 3000))) for _ in range(8)]
    units += [text[rng.randint(0, 10000):][:rng.randint(1, 9000)] for _ in range(30)]
    expected = [oc.bzip2_compress(u, k)[1] for u in units]
    in_buf, in_offs, _ = H.pack_hostile(units, rng)
    out_off, out_cap, pos = [], [], 7
    for j, e in enumerate(expected):
        d = j % 31 - 15
        cap = max(len(e) + d, 0)
        out_off.append(pos); out_cap.append(cap)
        pos += cap + 1 + j % 5
    st, ln, out = run_batch(units, in_offs, in_buf, out_off, out_cap, pos + 64, k, scratch)
    touched = np.zeros(len(out), dtype=bool)
    for j, e in enumerate(expected):
        assert ln[j] == len(e), j
        if out_cap[j] < len(e):
            assert st[j] == 1                                            # SWC_ERR_OUTPUT_OVERFLOW, nothing written
        else:
            assert st[j] == 0 and bytes(out[out_off[j]:out_off[j] + len(e)]) == e, j
            touched[out_off[j]:out_off[j] + len(e)] = True
    assert (out[~touched] == 0xA5).all()
    return st, ln, out


def test_batch_fenced(gpu, oc):
    fenced(oc)


def test_batch_fenced_in_slices(gpu, oc):
    """a 6 MiB caller scratch holds the largest unit (two blocks, about 3.5 MiB) but not the batch, which then runs in
    slices: the results must not change"""
    from swcompression_b200 import _lib
    assert _lib.lib().swc_bzip2_compress_batch_scratch_bytes(45, 300000, 1) > 6 << 20
    a = fenced(oc)
    b = fenced(oc, scratch=6 << 20)
    for x, y in zip(a, b):
        assert (x == y).all()


def test_scratch_bytes_run_one_slice(gpu, oc):
    """swc_bzip2_compress_batch_scratch_bytes is enough for one slice, also for batches of tiny units: one slice is
    9 kernel launches"""
    from swcompression_b200 import _lib
    L = _lib.lib()
    rng = random.Random(23)
    for units in ([bytes(rng.getrandbits(8) for _ in range(rng.randint(0, 84))) for _ in range(300)],
                  [b"x"] * 50 + [H.textlike(80001, 3)] + [bytes(200)] * 50):
        expected = [oc.bzip2_compress(u, 1)[1] for u in units]
        in_buf, in_offs, _ = H.pack_hostile(units, rng)
        out_off = np.cumsum([0] + [len(e) + 3 for e in expected[:-1]]) + 5
        before = L.swc_kernel_launches()
        st, ln, out = run_batch(units, in_offs, in_buf, out_off, [len(e) for e in expected], int(out_off[-1]) + len(expected[-1]) + 64, 1)
        assert L.swc_kernel_launches() - before == 9
        for j, e in enumerate(expected):
            assert st[j] == 0 and bytes(out[out_off[j]:out_off[j] + len(e)]) == e, j


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
