"""Parity of the CUDA Deflate path (through the C ABI) with the CPU oracle: golden fixtures, the reference's inline
malformed vectors, round trips, batched synthetic corpora (BASELINE config 1/2 shape), edge cases and truncation fuzz."""
import random
import zlib

import numpy as np
import pytest

import helpers as H

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def gpu():
    import torch
    assert torch.cuda.is_available()
    import swcompression_b200 as S
    return S


def run_batch(units, cap):
    from swcompression_b200.batch import Batch
    b = Batch.from_units("deflate", units, cap)
    b.run()
    st, ln, used = b.results()
    return st, ln, used, b.outputs()


def same_as_oracle(oracle, units, cap):
    st, ln, used, outs = run_batch(units, cap)
    caps = np.full(len(units), cap) if np.isscalar(cap) else cap
    for i, u in enumerate(units):
        ost, oout, oused = oracle.deflate_decompress(u)
        if ost == 0 and len(oout) > caps[i]:
            assert st[i] == 1 and ln[i] == len(oout), (i, st[i], ln[i], len(oout))     # overflow reports the needed size
        elif ost == 0:
            assert st[i] == 0 and outs[i] == oout and used[i] == oused, (i, st[i], ost)
        else:
            assert st[i] == ost, (i, st[i], ost)


@pytest.mark.parametrize("rel,ans", H.fixtures("Deflate/"))
def test_fixture(gpu, rel, ans):
    assert gpu.Deflate.decompress(H.fixture(rel)) == H.answer(ans)


def test_inline_vectors(gpu, oracle):
    from test_oracle_golden import DEFLATE_INLINE
    for data, expect in DEFLATE_INLINE:
        ost = oracle.deflate_decompress(data)[0]
        if expect is None:
            with pytest.raises(gpu.SWCompressionError) as e:
                gpu.Deflate.decompress(data)
            assert e.value.code == ost
        else:
            assert gpu.Deflate.decompress(data) == expect


@pytest.mark.parametrize("raw", H.ROUNDTRIP_STRINGS)
def test_roundtrip_strings(gpu, raw):
    for lvl in (0, 1, 6, 9):
        assert gpu.Deflate.decompress(H.raw_deflate(raw, lvl, 8)) == raw


def test_config1_single_dynamic_block(gpu, oracle):
    raw = H.textlike(65536, 1)
    comp = H.raw_deflate(raw)
    assert comp[0] & 7 == 0b101, "BASELINE config 1 must be ONE final dynamic-Huffman block"
    out, used = gpu.Deflate.decompress_from(comp, 0)
    ost, oout, oused = oracle.deflate_decompress(comp)
    assert ost == 0 and out == oout == raw and used == oused and (used + 7) // 8 == len(comp)


def test_batch_textlike_64k(oracle):
    raws = [H.textlike(65536, 2 + i) for i in range(300)]
    units = [H.raw_deflate(r) for r in raws]
    same_as_oracle(oracle, units, 65536)


def test_batch_ragged_and_mixed_block_types(oracle):
    rng = random.Random(5)
    units = []
    for i in range(200):
        n = rng.choice([0, 1, 2, 7, 8, 9, 15, 16, 17, 100, 1000, 5000, 70000, 200000])
        kind = rng.randrange(4)
        if kind == 0:
            raw = H.textlike(max(n, 70), i)[:n]
        elif kind == 1:
            raw = bytes(rng.getrandbits(8) for _ in range(n))            # incompressible -> stored blocks
        elif kind == 2:
            raw = bytes(n)                                               # long overlapping matches (dist 1)
        else:
            raw = (b"abc" * (n // 3 + 1))[:n]
        lvl = rng.choice([0, 1, 6, 9])
        strategy = rng.choice([zlib.Z_DEFAULT_STRATEGY, zlib.Z_FIXED, zlib.Z_HUFFMAN_ONLY, zlib.Z_RLE])
        c = zlib.compressobj(lvl, zlib.DEFLATED, -15, rng.choice([1, 8, 9]), strategy)
        data = c.compress(raw[:n // 2]) + c.flush(zlib.Z_FULL_FLUSH if i % 3 == 0 else zlib.Z_NO_FLUSH) + c.compress(raw[n // 2:]) + c.flush()
        units.append(data)
    same_as_oracle(oracle, units, 200000)


def test_overflow_reports_required_size(oracle):
    raws = [H.textlike(30000 + 977 * i, 40 + i) for i in range(40)]
    units = [H.raw_deflate(r) for r in raws]
    caps = np.array([len(r) - (i % 5) * 1000 for i, r in enumerate(raws)], dtype=np.uint64)
    same_as_oracle(oracle, units, caps)


def test_truncation_and_corruption_fuzz(oracle):
    rng = random.Random(11)
    base = [H.raw_deflate(H.textlike(20000, 70)), H.raw_deflate(H.textlike(3000, 71), 0),
            zlib.compressobj(6, zlib.DEFLATED, -15, 8, zlib.Z_FIXED).compress(H.textlike(5000, 72))]
    c = zlib.compressobj(6, zlib.DEFLATED, -15, 8, zlib.Z_FIXED)
    base[2] = c.compress(H.textlike(5000, 72)) + c.flush()
    units = []
    for d in base:
        for _ in range(60):
            units.append(d[:rng.randrange(1, len(d))])
        for _ in range(60):
            b = bytearray(d)
            for _ in range(rng.randrange(1, 4)):
                b[rng.randrange(len(b))] ^= 1 << rng.randrange(8)
            units.append(bytes(b))
    st, ln, used, outs = run_batch(units, 1 << 20)
    for i, u in enumerate(units):
        ost, oout, oused = oracle.deflate_decompress(u)
        assert st[i] == ost, (i, st[i], ost)
        if ost == 0:
            assert outs[i] == oout and used[i] == oused


def test_malformed_huffman_sets_match_reference_semantics(oracle):
    # bit flips inside dynamic-block headers produce incomplete and OVER-SUBSCRIBED code sets; the reference accepts
    # both (heap-slot overwrite semantics, DecodingTree.swift:15-50). Over-subscribed sets take the generic decoder.
    rng = random.Random(13)
    units = []
    for seed in range(6):
        d = H.raw_deflate(H.textlike(3000 + seed * 500, 80 + seed))
        for _ in range(120):
            b = bytearray(d)
            for _ in range(rng.randrange(1, 3)):
                b[rng.randrange(min(len(b), 70))] ^= 1 << rng.randrange(8)
            units.append(bytes(b))
    st, ln, used, outs = run_batch(units, 1 << 20)
    ok = 0
    for i, u in enumerate(units):
        ost, oout, oused = oracle.deflate_decompress(u)
        assert st[i] == ost, (i, st[i], ost)
        if ost == 0:
            ok += 1
            assert outs[i] == oout and used[i] == oused
    assert ok > 0


def test_start_bit_form(gpu, oracle):
    raw = H.textlike(5000, 9)
    comp = H.raw_deflate(raw)
    w = H.LsbBitWriter()
    w.write_number(0b10110, 5)                    # 5 junk bits before the stream
    for byte in comp:
        w.write_number(byte, 8)
    data = b"\xAA\xBB" + w.data
    out, used = gpu.Deflate.decompress_from(data, 16 + 5)
    ost, oout, oused = oracle.deflate_decompress(data, 16 + 5)
    assert ost == 0 and out == oout == raw and used == oused


def test_batch_host_pipelined(oracle):
    """swc_deflate_decompress_batch_host: host buffers in/out, sliced over three streams when n >= 4096."""
    import ctypes as C
    from swcompression_b200 import _lib
    from swcompression_b200.batch import pack_units
    base = [H.raw_deflate(H.textlike(4000 + 37 * i, 3000 + i)) for i in range(64)]
    raws = [H.textlike(4000 + 37 * i, 3000 + i) for i in range(64)]
    for n in (100, 5000):
        units = [base[i % 64] for i in range(n)]
        buf, offs, lens = pack_units(units)
        cap = 8192
        o_off = np.arange(n, dtype=np.uint64) * np.uint64(cap)
        o_cap = np.full(n, cap, dtype=np.uint64)
        out = np.zeros(n * cap, dtype=np.uint8)
        r_len = np.zeros(n, dtype=np.uint64); r_used = np.zeros(n, dtype=np.uint64); r_st = np.full(n, -1, dtype=np.int32)
        vp = lambda a: a.ctypes.data_as(C.c_void_p)
        rc = _lib.lib().swc_deflate_decompress_batch_host(vp(buf), vp(offs), vp(lens), len(buf), vp(out), vp(o_off), vp(o_cap), n * cap,
                                                         vp(r_len), vp(r_used), vp(r_st), n)
        assert rc == 0
        assert (r_st == 0).all()
        for i in range(0, n, 97):
            ost, oout, oused = oracle.deflate_decompress(units[i])
            assert bytes(out[i * cap:i * cap + int(r_len[i])]) == oout == raws[i % 64] and r_used[i] == oused


def test_large_batch_thread_kernel(oracle):
    """>= 20000 units take K1L, the thread-per-unit table-lookup decoder (inflate_lut.cu; persistent lanes, ticket
    counter): valid, stored, truncated, corrupted, over-subscribed (slow kernel) and empty units side by side, all equal
    to the oracle."""
    rng = random.Random(17)
    distinct = []
    for i in range(40):
        distinct.append(H.raw_deflate(H.textlike(rng.randrange(200, 9000), 300 + i), rng.choice((1, 6, 9))))
    distinct.append(H.raw_deflate(H.textlike(4000, 350), 0))                     # stored blocks
    distinct.append(H.raw_deflate(b""))
    distinct.append(H.raw_deflate(bytes(7000)))                                  # one long overlapping match chain
    good = list(distinct)
    for d in good[:12]:
        distinct.append(d[:rng.randrange(1, len(d))])                             # truncated
        b = bytearray(d)
        b[rng.randrange(min(len(b), 60))] ^= 1 << rng.randrange(8)                # damaged header / early payload
        distinct.append(bytes(b))
    expect = [oracle.deflate_decompress(u) for u in distinct]
    n = 24576
    order = [rng.randrange(len(distinct)) for _ in range(n)]
    st, ln, used, outs = run_batch([distinct[i] for i in order], 16384)
    for j, i in enumerate(order):
        ost, oout, oused = expect[i]
        if ost == 0 and len(oout) > 16384:
            assert st[j] == 1 and ln[j] == len(oout)
        elif ost == 0:
            assert st[j] == 0 and outs[j] == oout and used[j] == oused, (j, i, st[j])
        else:
            assert st[j] == ost, (j, i, st[j], ost)


def test_benched_config_lut_kernel_all_units(oracle):
    """BASELINE configs[1] shape through the kernels bench.py times: >= 20 000 units of 65 536-byte single dynamic-Huffman
    blocks take the thread-per-unit table-lookup decoder (inflate_lut.cu) + the record-replay kernel.  Every one of the
    512 distinct units is compared byte for byte (and its consumed bit count) with the oracle, and every tiled copy with the
    first copy on the device."""
    import torch
    from swcompression_b200.batch import Batch, pack_units
    distinct, tile = 512, 40
    raws = [H.textlike(65536, 5000 + i) for i in range(distinct)]
    units = [H.raw_deflate(r) for r in raws]
    assert all(u[0] & 7 == 0b101 for u in units)
    buf, offs, lens = pack_units(units)
    stride = len(buf) - 64
    big = np.concatenate([np.tile(buf[:stride], tile), np.zeros(64, dtype=np.uint8)])
    all_off = (offs[None, :] + (np.arange(tile, dtype=np.uint64) * np.uint64(stride))[:, None]).reshape(-1)
    all_len = np.tile(lens, tile)
    b = Batch("deflate", big, all_off, all_len, 65536)
    assert b.n == distinct * tile >= 20000
    b.run()
    st, ln, used = b.results()
    assert (st == 0).all() and (ln == 65536).all()
    out = b.d_out[: b.n * 65536].view(tile, distinct, 65536)
    assert bool((out == out[0:1]).all()), "tiled copies differ"
    first = out[0].cpu().numpy()
    for i, u in enumerate(units):
        ost, oout, oused = oracle.deflate_decompress(u)
        assert ost == 0 and bytes(first[i]) == oout == raws[i], i
        assert (used[i::distinct] == oused).all(), i
