"""The CUDA LZ4 compressor (lz4_compress.cu through swc_lz4_compress / swc_lz4_block_compress_batch) byte for byte
against the CPU restatement of LZ4+Compress.swift, and back through the GPU decoder."""
import random

import numpy as np
import pytest

import compress_batch as CB
import helpers as H
import lz4c_cases as K

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def oc():
    """the CPU restatement of LZ4+Compress.swift (oracle/swco_lz4c.py)"""
    import swco_lz4c
    swco_lz4c.lib()
    return swco_lz4c


@pytest.fixture(scope="module")
def gpu():
    import torch
    assert torch.cuda.is_available()
    import swcompression_b200 as S
    return S


def check_frame(S, oc, data, **opts):
    st, expected, _ = oc.lz4_compress(data, **opts)
    assert st == 0
    got = S.LZ4.compress(data, **opts)
    assert got == expected, (len(data), opts)
    d = opts.get("dictionary")
    if opts.get("dictionaryID") is not None and d is None:
        d = b""                                   # the decoder wants a dictionary whenever the frame names one
    assert S.LZ4.decompress(got, dictionary=d) == data


@pytest.mark.parametrize("data", K.STRINGS + [K.TRICKY], ids=lambda d: d[:12].hex())
def test_reference_strings(gpu, oc, data):
    check_frame(gpu, oc, data)
    assert gpu.LZ4.compress(data) == oc.lz4_compress(data)[1]


def test_tricky_sequence(gpu, oc):
    check_frame(gpu, oc, K.TRICKY, **K.TRICKY_OPTS)


@pytest.mark.parametrize("name", ["test1", "test5", "test6", "zeros5m"])
def test_answers(gpu, oc, name):                            # LZ4CompressionTests.swift:50-84
    check_frame(gpu, oc, H.answer(name))


@pytest.mark.parametrize("name,block,dictionary,variant", K.edge_blocks(), ids=lambda v: v if isinstance(v, str) else None)
def test_edge_blocks_in_frames(gpu, oc, name, block, dictionary, variant):
    opts = dict(independentBlocks=True, blockChecksums=True, contentChecksum=True, contentSize=True)
    if dictionary:
        opts["dictionary"] = dictionary
    check_frame(gpu, oc, block, **opts)


def test_incompressible_and_equal_size(gpu, oc):
    rng = random.Random(11)
    for n in (1, 13, 100, 4097, 65536, 300000):
        check_frame(gpu, oc, bytes(rng.getrandbits(8) for _ in range(n)), blockSize=65536, blockChecksums=True)
    eq = K.compressible_equal_size()
    check_frame(gpu, oc, eq)
    assert gpu.LZ4.compress(eq)[11:11 + len(eq)] != eq           # kept compressed although no shorter


def test_dictionaries(gpu, oc):
    small = H.fixture("LZ4/lz4_small_dict")
    text = dict(K.frame_inputs())["text"]
    rng = random.Random(2)
    big = bytes(rng.getrandbits(8) for _ in range(30000)) + text[:50000]
    for d in (small, big, text[:4], b""):
        for independent in (True, False):
            check_frame(gpu, oc, text, independentBlocks=independent, blockChecksums=True, contentChecksum=True,
                        contentSize=False, blockSize=256 * 1024 if d is small else 65536, dictionary=d)
    check_frame(gpu, oc, text[:5000], independentBlocks=True, blockChecksums=False, contentChecksum=True,
                contentSize=True, dictionary=small, dictionaryID=20000)
    check_frame(gpu, oc, text[:5000], independentBlocks=True, blockChecksums=False, contentChecksum=True,
                contentSize=True, dictionaryID=7)


@pytest.mark.parametrize("kwargs", [dict(blockSize=0), dict(blockSize=-5), dict(blockSize=(4 << 20) + 1),
                                    dict(dictionary=b"a"), dict(dictionary=b"ab"), dict(dictionary=b"abc"),
                                    dict(independentBlocks=False, blockSize=3), dict(independentBlocks=False, blockSize=2)])
def test_reference_traps(gpu, oc, kwargs):
    assert oc.lz4_compress(b"abcdefgh", **kwargs)[0] == 2
    with pytest.raises(gpu.EngineError) as e:
        gpu.LZ4.compress(b"abcdefgh", **kwargs)
    assert e.value.case == "referenceTrap"
    assert gpu.LZ4.compress(b"", dictionary=b"ab") == oc.lz4_compress(b"", dictionary=b"ab")[1]


@pytest.mark.parametrize("bs", K.SWEEP_BLOCK_SIZES)
def test_option_sweep(gpu, oc, bs):
    for name, data in K.frame_inputs():
        for ind in (True, False):
            for bc in (False, True):
                for cc in (False, True):
                    for cs in (False, True):
                        if bs == 1024 and len(data) > 80000 and (bc, cc, cs) != (True, True, True):
                            continue                               # keep the 1 KiB x 150 KB frames to one combination
                        check_frame(gpu, oc, data, independentBlocks=ind, blockChecksums=bc, contentChecksum=cc,
                                    contentSize=cs, blockSize=bs)


# ---- the batched raw form: the layout and slice contract it shares with Deflate and BZip2 (compress_batch.py) ----------

def test_batch_unaligned_fenced(gpu):
    CB.one_slice("lz4_block_compress")


def test_batch_fenced_in_slices(gpu):
    CB.in_slices("lz4_block_compress")


def test_scratch_bytes_run_one_slice(gpu):
    CB.tiny_units_one_slice("lz4_block_compress")


def test_scratch_below_largest_unit_is_invalid(gpu):
    CB.below_largest_unit_is_invalid("lz4_block_compress")


def test_batch_dictionary_windows(gpu, oc):
    """both frame modes as windows into the input: the previous block's last 64 KiB, and one shared user dictionary"""
    text = dict(K.frame_inputs())["text"] * 2
    small = H.fixture("LZ4/lz4_small_dict")
    buf = small + text
    bs = 40000
    units, in_offs, d_off, d_len, dicts = [], [], [], [], []
    for o in range(0, len(text), bs):
        blk = text[o:o + bs]
        units.append(blk); in_offs.append(len(small) + o)
        if o == 0:
            d_off.append(0); d_len.append(len(small)); dicts.append(small)
        else:
            w = min(bs, 65536)
            d_off.append(len(small) + o - w); d_len.append(w); dicts.append(text[o - w:o])
    units.append(text[:3000]); in_offs.append(len(small)); d_off.append(0); d_len.append(len(buf)); dicts.append(buf)
    units.append(text[:100]); in_offs.append(len(small)); d_off.append(0); d_len.append(2); dicts.append(buf[:2])
    from swcompression_b200.batch import Batch
    in_buf = np.frombuffer(buf + bytes(64), dtype=np.uint8).copy()
    b = Batch("lz4_block_compress", in_buf, in_offs, [len(u) for u in units], [len(u) + len(u) // 200 + 64 for u in units],
              aux=(d_off, d_len))
    b.run()
    st, ln, _ = b.results()
    outs = b.outputs()
    for k, (u, d) in enumerate(zip(units, dicts)):
        ost, exp, _ = oc.lz4_block_compress(u, d)
        assert st[k] == ost, k
        if ost == 0:
            assert ln[k] == len(exp) and outs[k] == exp, k
    assert st[-1] == 2


def test_benched_shape(gpu, oc):
    """20 480 tiled units of the benchmark's mix: every copy equals the first on the device, the distinct ones the oracle"""
    import torch
    from swcompression_b200.batch import Batch
    rng = random.Random(4)
    distinct = []
    for i in range(64):
        r = i % 10
        distinct.append(bytes(65536) if r == 8 else bytes(rng.getrandbits(8) for _ in range(65536)) if r == 9
                        else H.textlike(65536, 500 + i))
    tile = 320
    buf = np.frombuffer(b"".join(distinct) * tile + bytes(64), dtype=np.uint8)
    offs = np.arange(64 * tile, dtype=np.uint64) * np.uint64(65536)
    b = Batch("lz4_block_compress", buf, offs, np.full(64 * tile, 65536, dtype=np.uint64), 65536 + 65536 // 255 + 64)
    b.run()
    st, ln, _ = b.results()
    assert (st == 0).all()
    assert (ln.reshape(tile, 64) == ln[:64][None, :]).all()
    cap = int(b.h_out_cap[0] + 15) // 16 * 16
    out = b.d_out[: 64 * tile * cap].view(tile, 64, cap)
    first = out[0:1]
    for k in range(64):
        L = int(ln[k])
        assert bool((out[:, k, :L] == first[:, k, :L]).all()), k
    host = first[0].cpu().numpy()
    for k, u in enumerate(distinct):
        assert bytes(host[k, :int(ln[k])]) == oc.lz4_block_compress(u)[1], k
    del out, first, b
    torch.cuda.empty_cache()
