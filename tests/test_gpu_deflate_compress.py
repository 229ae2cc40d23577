"""The CUDA Deflate compressor (deflate_compress.cu through swc_deflate_compress_batch and the single calls) byte for
byte against the CPU restatement of Deflate+Compress.swift, GzipArchive.archive and ZlibArchive.archive, and back
through the engine's own decoders."""
import ctypes as C
import random
import struct

import numpy as np
import pytest

import compress_batch as CB
import deflatec_cases as K
import helpers as H

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def oc():
    import swco_deflatec
    swco_deflatec.lib()
    return swco_deflatec


@pytest.fixture(scope="module")
def gpu():
    import torch
    assert torch.cuda.is_available()
    import swcompression_b200 as S
    return S


def bound(n):
    return (9 * n + 17) // 8


def test_catalogue_and_answers_batch(gpu, oc):
    from swcompression_b200.batch import Batch
    units = [d for _, d in K.cases()] + [H.answer(a) for a in ("test1", "test5", "test6", "zeros5m")]
    b = Batch.from_units("deflate_compress", units, [bound(len(u)) for u in units])
    b.run()
    st, ln, _ = b.results()
    outs = b.outputs()
    for k, u in enumerate(units):
        ost, exp, _ = oc.deflate_compress(u)
        assert st[k] == ost == 0 and ln[k] == len(exp) and outs[k] == exp, k
    # round trip through the engine's own batch decoder
    d = Batch.from_units("deflate", outs, [max(len(u), 16) for u in units])
    d.run()
    dst, dln, _ = d.results()
    assert (dst == 0).all() and d.outputs() == units


def test_single_calls(gpu, oc):
    S = gpu
    for data in [H.textlike(64 << 20, 5), bytes(64 << 20), np.random.default_rng(3).bytes(16 << 20)]:
        got = S.Deflate.compress(data)
        assert got == oc.deflate_compress(data)[1], len(data)
        assert S.Deflate.decompress(got) == data


def test_archives_option_grid(gpu, oc):
    S = gpu
    data = H.textlike(300000, 11)
    z = S.ZlibArchive.archive(data)
    assert z == oc.zlib_archive(data)[1] and S.ZlibArchive.unarchive(z) == data
    assert S.ZlibArchive.archive(b"") == oc.zlib_archive(b"")[1]
    osn = {"fat": 0, "unix": 3, "macintosh": 7, "ntfs": 11, "other": 255, None: 255}
    rng = random.Random(2)
    for comment in (None, "", "comment \xe9", "z\0"):
        for name in (None, "file.txt"):
            for hcrc in (False, True):
                for os in osn:
                    mt = rng.choice([None, 0, -1.5, 1700000000.75, 2**40 + 5])
                    tx = rng.random() < 0.5
                    ex = rng.choice([[], [S.ExtraField(65, 66, b"")], [S.ExtraField(1, 2, b"xy"), S.ExtraField(3, 4, bytes(300))]])
                    got = S.GzipArchive.archive(data, comment=comment, fileName=name, writeHeaderCRC=hcrc, isTextFile=tx,
                                                osType=os, modificationTime=mt, extraFields=ex)
                    exp = oc.gzip_archive(data, comment=None if comment is None else comment.encode("latin-1"),
                                          fileName=None if name is None else name.encode("latin-1"), writeHeaderCRC=hcrc,
                                          isTextFile=tx, osByte=osn[os], modificationTime=None if mt is None else int(mt),
                                          extraFields=[(e.si1, e.si2, e.bytes) for e in ex])[1]
                    assert got == exp, (comment, name, hcrc, os, mt)
    assert S.GzipArchive.unarchive(got) == data


def test_gzip_errors(gpu):
    S = gpu
    from swcompression_b200.errors import GzipError
    with pytest.raises(GzipError) as e:
        S.GzipArchive.archive(b"x", comment="€")
    assert e.value.code == 607
    with pytest.raises(GzipError) as e:
        S.GzipArchive.archive(b"x", extraFields=[S.ExtraField(1, 1, bytes(65532))])
    assert e.value.code == 607
    ok = S.GzipArchive.archive(b"x", extraFields=[S.ExtraField(1, 1, bytes(65531))])
    assert S.GzipArchive.unarchive(ok) == b"x"


# ---- the batch layout and slice contract it shares with LZ4 and BZip2 (compress_batch.py) ------------------------------

def test_batch_fenced(gpu):
    CB.one_slice("deflate_compress")


def test_batch_fenced_in_slices(gpu):
    CB.in_slices("deflate_compress")


def test_scratch_bytes_run_one_slice(gpu):
    CB.tiny_units_one_slice("deflate_compress")


def test_scratch_below_largest_unit_is_invalid(gpu):
    CB.below_largest_unit_is_invalid("deflate_compress")


def test_benched_shape_and_bgzf_round_trip(gpu, oc):
    """20 480 tiled units of the benchmark's mix; then a BGZF-shaped archive of the distinct outputs, CRC-32 on device"""
    import torch
    from swcompression_b200 import _lib
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
    b = Batch("deflate_compress", buf, offs, np.full(64 * tile, 65536, dtype=np.uint64), bound(65536))
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
    streams = [bytes(host[k, :int(ln[k])]) for k in range(64)]
    for k, u in enumerate(distinct):
        assert streams[k] == oc.deflate_compress(u)[1], k
    del out, first
    # CRC-32 of the 64 distinct inputs on the device, then gzip members around the batch's streams
    dev = torch.device("cuda:0")
    d_in = b.d_in
    d_off = torch.from_numpy((np.arange(64, dtype=np.uint64) * np.uint64(65536)).view(np.int64)).to(dev)
    d_len = torch.full((64,), 65536, dtype=torch.int64, device=dev)
    d_crc = torch.zeros(64, dtype=torch.int32, device=dev)
    assert _lib.lib().swc_crc32_batch(C.c_void_p(d_in.data_ptr()), C.c_void_p(d_off.data_ptr()), C.c_void_p(d_len.data_ptr()),
                                      None, C.c_void_p(d_crc.data_ptr()), 64,
                                      C.c_void_p(torch.cuda.current_stream(dev).cuda_stream)) == 0
    crcs = d_crc.cpu().numpy().view(np.uint32)
    archive = b"".join(b"\x1f\x8b\x08\x00\x00\x00\x00\x00\x02\xff" + s + struct.pack("<II", int(c), 65536)
                       for s, c in zip(streams, crcs))
    members = gpu.GzipArchive.multiUnarchive(archive)
    assert [m.data for m in members] == distinct
    del b
    torch.cuda.empty_cache()
