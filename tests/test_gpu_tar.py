"""swc_tar_walk_batch and the single TarContainer calls against the CPU restatement (oracle/tar.c): the whole catalogue,
every byte cut of the small cases, hostile layouts, entry-table overflow, a gzip -> tar chain, a CUDA graph, and an
archive whose last header lies past 4 GiB."""
import gzip

import numpy as np
import pytest
import torch

import swco_tar
import tar_cases as T
import tar_writer as W
from swcompression_b200 import TarContainer, TarError, EngineError
from swcompression_b200.api import tar_entry, tar_entry_info
from swcompression_b200.batch import Batch

pytestmark = pytest.mark.gpu
CASES = T.cases()
FORMATS = ["prePosix", "ustar", "gnu", "pax"]


def _check_batch(b, units, caps=None):
    n, ist, ost, fmt, fst = b.tar_results()
    for i, data in enumerate(units):
        cap = int(b.h_entry_cap[i])
        on, oi, oo, of, ofs, recs = swco_tar.walk(data, cap=cap)
        assert (int(n[i]), int(ist[i]), int(ost[i]), int(fst[i])) == (on, oi, oo, ofs), f"unit {i}"
        if ofs == 0:
            assert int(fmt[i]) == of, f"unit {i}"
        assert b.records(i) == recs, f"unit {i}"


def test_batch_catalogue():
    units = [c[1] for c in CASES]
    b = Batch.from_units("tar", units, None)
    b.run()
    _check_batch(b, units)
    for i, c in enumerate(CASES):
        assert int(b.tar_results()[1][i]) == c[2], c[0]


def _expect(fn, data, walked=None):
    n, ist, ost, fmt, fst, recs = walked or swco_tar.walk(data)
    if fn == "info":
        return ist, [tar_entry_info(data, r) for r in recs]
    if fn == "open":
        return ost, [tar_entry(data, r) for r in recs]
    return fst, FORMATS[fmt]


def _same(a, b):
    return a == b or repr(a) == repr(b)                           # NaN times compare by repr


def _check_single(data):
    walked = swco_tar.walk(data)
    for fn in ("info", "open", "formatOf"):
        st, want = _expect(fn if fn != "formatOf" else "format", data, walked)
        if st == 0:
            assert _same(getattr(TarContainer, fn)(data), want), fn
        else:
            with pytest.raises((TarError, EngineError)) as ei:
                getattr(TarContainer, fn)(data)
            assert ei.value.code == st, fn


@pytest.mark.parametrize("case", CASES, ids=[c[0] for c in CASES])
def test_single_calls(case):
    _check_single(case[1])


@pytest.mark.parametrize("cid", T.SMALL_CUTS)
def test_every_cut_single_calls(cid):
    data = {c[0]: c[1] for c in CASES}[cid]
    for m in range(len(data) + 1):
        _check_single(data[:m])


def test_every_cut():
    byid = {c[0]: c[1] for c in CASES}
    units = [byid[k][:m] for k in T.SMALL_CUTS for m in range(len(byid[k]) + 1)]
    b = Batch.from_units("tar", units, None)
    b.run()
    _check_batch(b, units)


def test_unaligned_back_to_back():
    units = [c[1] for c in CASES if len(c[1]) < 20000]
    for shift in (1, 7, 13):
        blob = b"\xee" * shift + b"".join(units) + b"\xee" * 64
        offs = np.cumsum([shift] + [len(u) for u in units[:-1]]).astype(np.uint64)
        lens = np.array([len(u) for u in units], dtype=np.uint64)
        b = Batch("tar", np.frombuffer(blob, dtype=np.uint8), offs, lens, None)
        b.run()
        _check_batch(b, units)


def test_overflow_and_rerun():
    byid = {c[0]: c[1] for c in CASES}
    units = [byid[k] for k in ("types", "pax_global_persists", "negative_moves_back", "tarfile_pax", "empty")]
    b = Batch.from_units("tar", units, 1)
    b.run()
    n, ist, ost, _, _ = b.tar_results()
    for i, u in enumerate(units):
        full = swco_tar.walk(u)
        assert int(n[i]) == full[0]
        if full[0] > 1:
            assert int(ist[i]) == 1 and int(ost[i]) == (1 if full[2] == 0 else full[2])
    _check_batch(b, units)
    b2 = Batch.from_units("tar", units, np.maximum(n, 1).astype(np.uint64))
    b2.run()
    _check_batch(b2, units)
    assert (b2.tar_results()[1] == np.array([swco_tar.walk(u)[1] for u in units])).all()


def test_gzip_then_tar_same_stream():
    units = [d for cid, d, _ in T.tarfile_archives()] + [c[1] for c in CASES[:20]]
    gz = [gzip.compress(u, mtime=0) for u in units]
    g = Batch.from_units("gzip", gz, max(len(u) for u in units) + 1024)
    t = Batch.tar_of(g)
    g.run()
    t.run()
    st, ln, _ = g.results()
    assert (st == 0).all() and [int(x) for x in ln] == [len(u) for u in units]
    _check_batch(t, units)


def test_gzip_failures_are_not_walked():
    """A 'tar' batch over a 'gzip' batch whose units overflow their capacity or fail: the walk reports the gzip status
    and reads nothing; with only the capacity bound, the overflowing unit (the last one, at the end of the output
    buffer) is walked over exactly its capacity."""
    byid = {c[0]: c[1] for c in CASES}
    units = [byid[k] for k in ("tarfile_pax", "pax_local", "types", "tarfile_gnu")]
    gz = [gzip.compress(u, mtime=0) for u in units]
    bad_crc = bytearray(gz[1])
    bad_crc[-8] ^= 0xFF                                           # CRC-32 in the trailer: GzipError.wrongCRC
    bad_magic = b"\x00" + gz[2][1:]                               # GzipError.wrongMagic
    gz = [gz[0], bytes(bad_crc), bad_magic, gz[3]]
    caps = np.array([len(units[0]) + 64, len(units[1]) + 64, len(units[2]) + 64, len(units[3]) // 2], dtype=np.uint64)
    g = Batch.from_units("gzip", gz, caps)
    t = Batch.tar_of(g)
    g.run()
    t.run()
    gst, gln, _ = g.results()
    assert int(gst[0]) == 0 and int(gst[1]) == 605 and int(gst[2]) == 601 and int(gst[3]) == 1
    assert int(gln[3]) == len(units[3]) > int(caps[3])
    n, ist, ost, fmt, fst = t.tar_results()
    for i in (1, 2, 3):
        assert (int(n[i]), int(ist[i]), int(ost[i]), int(fst[i]), int(fmt[i])) == (0, int(gst[i]), int(gst[i]), int(gst[i]), 0)
    on, oi, oo, of, ofs, recs = swco_tar.walk(units[0], cap=int(t.h_entry_cap[0]))
    assert (int(n[0]), int(ist[0]), int(ost[0]), int(fst[0]), int(fmt[0])) == (on, oi, oo, ofs, of) and t.records(0) == recs
    # the capacity bound alone: unit 3 is walked over the first caps[3] bytes of its region
    c = Batch.__new__(Batch)
    c.codec, c.device, c.n = "tar", g.device, g.n
    c._init_tar(g.d_out, g.d_out_off, g.d_out_len, g.h_out_cap // np.uint64(512) + np.uint64(1), g.d_out_cap, None)
    c.run()
    region = c.unit_bytes(3)
    assert len(region) == int(caps[3])
    _check_batch(c, [c.unit_bytes(i) for i in range(c.n)])


def test_graph_replay():
    byid = {c[0]: c[1] for c in CASES}
    a = [byid[k] for k in ("pax_local", "gnu_long_name", "one_file")]
    bb = [byid[k] for k in ("prefix", "types", "checksum_mismatch")]
    slot = (max(len(x) for x in a + bb) + 15) // 16 * 16              # every unit gets a slot the second set fits
    buf = np.zeros(3 * slot + 64, dtype=np.uint8)
    for i, u in enumerate(a):
        buf[i * slot:i * slot + len(u)] = np.frombuffer(u, dtype=np.uint8)
    offs = np.arange(3, dtype=np.uint64) * np.uint64(slot)
    b = Batch("tar", buf, offs, np.array([len(u) for u in a], dtype=np.uint64), slot // 512 + 1)
    stream = torch.cuda.Stream()
    with torch.cuda.stream(stream):
        b.run()                                                   # warm-up outside the capture
    torch.cuda.synchronize()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g, stream=stream):
        b.run()
    g.replay()
    _check_batch(b, a)
    # new archives in place: same offsets, new lengths
    host = b.d_in.cpu().numpy().copy()
    for i, u in enumerate(bb):
        host[i * slot:i * slot + len(u)] = np.frombuffer(u, dtype=np.uint8)
    b.d_in.copy_(torch.from_numpy(host))
    b.d_in_len.copy_(torch.tensor([len(u) for u in bb], dtype=torch.int64))
    g.replay()
    _check_batch(b, bb)


def test_header_past_4gib():
    gib4 = 4 << 30
    total = 512 + gib4 + 512 + 512 + 1024
    d = torch.zeros(total, dtype=torch.uint8, device="cuda:0")
    h1 = W.header(name=b"huge.bin", size=gib4)
    h2 = W.header(name=b"after", size=3)
    d[0:512] = torch.frombuffer(bytearray(h1), dtype=torch.uint8).cuda()
    d[512 + gib4:1024 + gib4] = torch.frombuffer(bytearray(h2), dtype=torch.uint8).cuda()
    d[1024 + gib4:1027 + gib4] = torch.tensor([1, 2, 3], dtype=torch.uint8)
    b = Batch.__new__(Batch)
    b.codec, b.device, b.n = "tar", torch.device("cuda:0"), 1
    b._init_tar(d, torch.zeros(1, dtype=torch.int64, device="cuda:0"), torch.tensor([total], dtype=torch.int64, device="cuda:0"), 4)
    b.run()
    n, ist, ost, fmt, fst = b.tar_results()
    assert (int(n[0]), int(ist[0]), int(ost[0]), int(fmt[0]), int(fst[0])) == (2, 0, 0, 1, 0)
    r = b.records(0)
    assert (r[0]["size"], r[1]["header_off"], r[1]["data_off"], r[1]["size"]) == (gib4, 512 + gib4, 1024 + gib4, 3)
    small = h2 + W.pad(b"\1\2\3") + W.EOF_MARKER
    want = swco_tar.walk(small)[5][0]
    got = dict(r[1])
    for k in ("header_off", "data_off", "name_off", "link_off", "uname_off", "gname_off"):
        got[k] -= 512 + gib4
    assert got == want
