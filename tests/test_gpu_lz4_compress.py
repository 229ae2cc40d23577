"""The CUDA LZ4 compressor (lz4_compress.cu through swc_lz4_compress / swc_lz4_block_compress_batch) byte for byte
against the CPU restatement of LZ4+Compress.swift, and back through the GPU decoder."""
import ctypes as C
import random

import numpy as np
import pytest

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


# ---- the batched raw form --------------------------------------------------------------------------------------------

def run_batch(units, in_offs, in_buf, out_off, out_cap, out_total, dict_off=None, dict_len=None, fill=0xA5):
    import torch
    from swcompression_b200 import _lib
    dev = torch.device("cuda:0")
    t = lambda a: torch.from_numpy(np.ascontiguousarray(np.asarray(a, dtype=np.uint64)).view(np.int64)).to(dev)
    n = len(units)
    d_in = torch.from_numpy(in_buf).to(dev)
    d_out = torch.full((out_total,), fill, dtype=torch.uint8, device=dev)
    lens = np.array([len(u) for u in units], dtype=np.uint64)
    d_len, d_st = torch.zeros(n, dtype=torch.int64, device=dev), torch.full((n,), -1, dtype=torch.int32, device=dev)
    window = int(lens.sum()) + (0 if dict_len is None else int(np.minimum(np.asarray(dict_len, dtype=np.uint64), 65536).sum()))
    L = _lib.lib()
    scr = torch.empty(L.swc_lz4_compress_batch_scratch_bytes(n, window), dtype=torch.uint8, device=dev)
    keep = [t(in_offs), t(lens), t(out_off), t(out_cap)] + ([t(dict_off), t(dict_len)] if dict_off is not None else [None, None])
    p = lambda x: None if x is None else C.c_void_p(x.data_ptr())
    st = L.swc_lz4_block_compress_batch(p(d_in), p(keep[0]), p(keep[1]), p(keep[4]), p(keep[5]), p(d_out), p(keep[2]),
                                        p(keep[3]), p(d_len), p(d_st), n, p(scr), scr.numel(),
                                        C.c_void_p(torch.cuda.current_stream(dev).cuda_stream))
    assert st == 0
    torch.cuda.synchronize()
    return d_st.cpu().numpy(), d_len.cpu().numpy(), d_out.cpu().numpy()


def test_batch_unaligned_fenced(gpu, oc):
    rng = random.Random(17)
    text = dict(K.frame_inputs())["text"]
    units = [b"", b"a", b"abcdabcdabcdabcd", text[:1000], bytes(5000), text[3:70000]]
    units += [bytes(rng.getrandbits(8) for _ in range(rng.randint(0, 3000))) for _ in range(10)]
    units += [text[rng.randint(0, 10000):][:rng.randint(1, 9000)] for _ in range(30)]
    expected = [oc.lz4_block_compress(u)[1] for u in units]
    # inputs back to back at odd offsets; outputs at every capacity residue with 0xA5 gaps between them
    in_offs, pos = [], 3
    for u in units:
        in_offs.append(pos)
        pos += len(u)
    in_buf = np.zeros(pos + 64, dtype=np.uint8)
    for u, o in zip(units, in_offs):
        in_buf[o:o + len(u)] = np.frombuffer(u, dtype=np.uint8)
    out_off, out_cap, pos = [], [], 5
    for k, e in enumerate(expected):
        cap = len(e) + k % 17 if k % 5 else max(len(e) - 1, 0)       # every fifth unit is one byte short
        out_off.append(pos); out_cap.append(cap)
        pos += cap + 7
    st, ln, out = run_batch(units, in_offs, in_buf, out_off, out_cap, pos + 64)
    touched = np.zeros(len(out), dtype=bool)
    for k, e in enumerate(expected):
        assert ln[k] == len(e), k
        if k % 5 == 0 and len(e) > 0:
            assert st[k] == 1                                            # SWC_ERR_OUTPUT_OVERFLOW, required size in out_len
        else:
            assert st[k] == 0 and bytes(out[out_off[k]:out_off[k] + len(e)]) == e, k
        touched[out_off[k]:out_off[k] + out_cap[k]] = True
    assert (out[~touched] == 0xA5).all()


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
    in_buf = np.frombuffer(buf + bytes(64), dtype=np.uint8).copy()
    caps = [len(u) + len(u) // 200 + 64 for u in units]
    offs = list(np.cumsum([0] + caps[:-1]))
    st, ln, out = run_batch(units, in_offs, in_buf, offs, caps, sum(caps) + 64, d_off, d_len)
    for k, (u, d) in enumerate(zip(units, dicts)):
        ost, exp, _ = oc.lz4_block_compress(u, d)
        assert st[k] == ost, k
        if ost == 0:
            assert ln[k] == len(exp) and bytes(out[offs[k]:offs[k] + ln[k]]) == exp, k
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
