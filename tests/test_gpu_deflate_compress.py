"""The CUDA Deflate compressor (deflate_compress.cu through swc_deflate_compress_batch and the single calls) byte for
byte against the CPU restatement of Deflate+Compress.swift, GzipArchive.archive and ZlibArchive.archive, and back
through the engine's own decoders."""
import ctypes as C
import random
import struct

import numpy as np
import pytest

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


def run_batch(units, in_offs, in_buf, out_off, out_cap, out_total, scratch=None, fill=0xA5):
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
    nb = L.swc_deflate_compress_batch_scratch_bytes(n, int(lens.sum())) if scratch is None else scratch
    scr = torch.empty(nb, dtype=torch.uint8, device=dev)
    keep = [t(in_offs), t(lens), t(out_off), t(out_cap)]
    p = lambda x: C.c_void_p(x.data_ptr())
    st = L.swc_deflate_compress_batch(p(d_in), p(keep[0]), p(keep[1]), p(d_out), p(keep[2]), p(keep[3]), p(d_len), p(d_st),
                                      n, p(scr), scr.numel(), C.c_void_p(torch.cuda.current_stream(dev).cuda_stream))
    assert st == 0
    torch.cuda.synchronize()
    return d_st.cpu().numpy(), d_len.cpu().numpy(), d_out.cpu().numpy()


def fenced(oc, scratch=None):
    rng = random.Random(17)
    text = H.textlike(200000, 21)
    units = [b"", b"a", b"abcabcabcabc", text[:1000], bytes(5000), text[3:70000], text[:K.TILE + 1], bytes(range(200, 256))]
    units += [bytes(rng.getrandbits(8) for _ in range(rng.randint(0, 3000))) for _ in range(10)]
    units += [text[rng.randint(0, 10000):][:rng.randint(1, 9000)] for _ in range(40)]
    expected = [oc.deflate_compress(u)[1] for u in units]
    in_offs, pos = [], 3
    for u in units:
        in_offs.append(pos)
        pos += len(u)
    in_buf = np.zeros(pos + 64, dtype=np.uint8)
    for u, o in zip(units, in_offs):
        in_buf[o:o + len(u)] = np.frombuffer(u, dtype=np.uint8)
    # capacities at every residue: exact, 1-15 short, 1-15 long; regions 16-aligned with 0xA5 gaps between them
    out_off, out_cap, pos = [], [], 16
    for k, e in enumerate(expected):
        d = k % 31 - 15
        cap = max(len(e) + d, 0)
        out_off.append(pos); out_cap.append(cap)
        pos += (cap + 15) // 16 * 16 + 16
    st, ln, out = run_batch(units, in_offs, in_buf, out_off, out_cap, pos + 64, scratch)
    touched = np.zeros(len(out), dtype=bool)
    for k, e in enumerate(expected):
        assert ln[k] == len(e), k
        if out_cap[k] < len(e):
            assert st[k] == 1                                            # SWC_ERR_OUTPUT_OVERFLOW, nothing written
        else:
            assert st[k] == 0 and bytes(out[out_off[k]:out_off[k] + len(e)]) == e, k
            touched[out_off[k]:out_off[k] + len(e)] = True
    assert (out[~touched] == 0xA5).all()
    return st, ln, out


def test_batch_fenced(gpu, oc):
    fenced(oc)


def test_batch_fenced_in_slices(gpu, oc):
    """a caller scratch that holds only a few units forces slices: the results must not change"""
    a = fenced(oc)
    b = fenced(oc, scratch=2 << 20)
    for x, y in zip(a, b):
        assert (x == y).all()


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
