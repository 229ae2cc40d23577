"""The batch layout contract (include/swcgpu.h, "Batch layout") on every batched entry point.  Units start at every byte
alignment, packed back to back or between non-zero filler; cut streams are followed in memory by their own rest and
front-cut ones preceded by their first bytes; Deflate units start 0..7 bits into their first byte; output regions take
capacities of every residue mod 16 (exact, short by 1..15, long by 1..15) inside a buffer filled with a sentinel.  The
reference for every unit is the oracle on the unit's own bytes: status, output length (on overflow the required size, or
a lower bound of it for BZip2 and LZMA), consumed bits or bytes and output bytes must agree, and no byte outside the output
regions may change."""
import copy
import ctypes as C
import os
import random
import subprocess
import sys
import zlib

import numpy as np
import pytest

import helpers as H

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _dev(a):
    import torch
    a = np.ascontiguousarray(a)
    return torch.from_numpy(a.view(np.int64) if a.dtype == np.uint64 else a).cuda()


def _p(t):
    return None if t is None else C.c_void_p(t.data_ptr())


def _stream():
    import torch
    return C.c_void_p(torch.cuda.current_stream().cuda_stream)


class Layout:
    """A hostile batch: the units packed by pack_hostile, fenced output regions sized from the oracle's answers."""

    def __init__(self, codec, oracle, units, seed, dictionary=None, residues=None):
        self.codec, self.units = codec, units
        cache = {}
        self.expect = []
        for u in units:
            key = (u.data, repr(u.aux))
            if key not in cache:
                cache[key] = H.layout_oracle(codec, oracle, u.data, u.aux, dictionary)
            self.expect.append(cache[key])
        rng = random.Random(seed)
        self.buf, self.offs, self.lens = H.pack_hostile([u.data for u in units], rng, [u.head for u in units],
                                                        [u.tail for u in units], residues)
        sizes = [len(e[1]) if e[0] == 0 else None for e in self.expect]
        spare = max([s for s in sizes if s is not None] + [0]) + 1024      # a damaged unit never overflows before its error
        self.out_off, self.out_cap, self.total = H.fenced_layout(sizes, spare)
        self.n = len(units)

    def friendly(self):
        """the same units and output regions, the input packed by batch.pack_units (16-byte aligned, zeros behind)"""
        from swcompression_b200.batch import pack_units
        f = copy.copy(self)
        f.buf, f.offs, f.lens = pack_units([u.data for u in self.units])
        return f

    def check(self, st, ln, used, out, consumed=True):
        # BZip2 and LZMA stop at the capacity, so on overflow their out_len is a lower bound of the size (swcgpu.h)
        exact = self.codec in ("deflate", "lz4_block")
        bad = []
        for i, (u, (ost, oout, oused)) in enumerate(zip(self.units, self.expect)):
            o, cap = int(self.out_off[i]), int(self.out_cap[i])
            if ost == 0 and u.raw is not None and oout != u.raw:
                bad.append((i, "oracle differs from the original bytes"))
            if ost == 0 and len(oout) > cap:
                if st[i] != 1 or (ln[i] != len(oout) if exact else ln[i] > len(oout)):
                    bad.append((i, "overflow", int(st[i]), int(ln[i]), len(oout)))
            elif ost == 0:
                if st[i] != 0 or ln[i] != len(oout):
                    bad.append((i, "status/length", int(st[i]), int(ln[i]), len(oout)))
                elif bytes(out[o:o + len(oout)]) != oout:
                    bad.append((i, "bytes"))
                elif consumed and used[i] != oused:
                    bad.append((i, "consumed", int(used[i]), oused))
            elif st[i] != ost and not (self.codec == "bzip2" and st[i] in (1, 6)):
                # (a damaged or cut BZip2 unit may instead hit the engine's documented limits, DESIGN.md §6: a corrupted run
                # length beyond the output bound, or an over-subscribed code set, which cut tables read as)
                bad.append((i, "status", int(st[i]), ost))
        fence = H.fence_violations(out, self.out_off, self.out_cap)
        assert not bad and fence.size == 0, (f"{self.codec}: {len(bad)} of {self.n} units differ from the oracle {bad[:8]}; "
                                             f"{fence.size} bytes changed outside the output regions, first at {fence[:8].tolist()}")


def run_both(lay, run, *args, **kw):
    """Run the hostile layout and the same units packed friendly.  The oracle says nothing about a failing unit's output
    length or consumed count, but those too must come from the unit's own bytes: every unit's status, out_len and
    consumed must be the same in both runs.  -> the hostile run's results"""
    a = run(lay, *args, **kw)
    b = run(lay.friendly(), *args, **kw)
    diff = np.nonzero((a[0] != b[0]) | (a[1] != b[1]) | (a[2] != b[2]))[0]
    assert diff.size == 0, (f"{lay.codec}: {diff.size} of {lay.n} units answer differently with foreign neighbours "
                            f"(index, status, out_len, consumed: hostile / friendly) "
                            f"{[(int(i), a[0][i], b[0][i], a[1][i], b[1][i], a[2][i], b[2][i]) for i in diff[:6]]}")
    return a


def _results(n):
    import torch
    return (torch.zeros(n, dtype=torch.int64, device="cuda"), torch.zeros(n, dtype=torch.int64, device="cuda"),
            torch.full((n,), -1, dtype=torch.int32, device="cuda"))


def _host(d_len, d_used, d_st, d_out):
    import torch
    torch.cuda.synchronize()
    return d_st.cpu().numpy(), d_len.cpu().numpy(), d_used.cpu().numpy(), d_out.cpu().numpy()


def run_deflate(lay, start_bits=None):
    import torch
    from swcompression_b200 import _lib
    L = _lib.lib()
    d_in, d_off, d_len = _dev(lay.buf), _dev(lay.offs), _dev(lay.lens)
    d_sb = None if start_bits is None else _dev(np.asarray(start_bits, dtype=np.uint8))
    d_ooff, d_ocap = _dev(lay.out_off), _dev(lay.out_cap)
    d_out = torch.full((lay.total,), H.SENTINEL, dtype=torch.uint8, device="cuda")
    r_len, r_used, r_st = _results(lay.n)
    scratch = torch.empty(L.swc_deflate_batch_scratch_bytes(lay.n, lay.total), dtype=torch.uint8, device="cuda")
    rc = L.swc_deflate_decompress_batch(_p(d_in), _p(d_off), _p(d_len), _p(d_sb), _p(d_out), _p(d_ooff), _p(d_ocap), lay.total,
                                        _p(r_len), _p(r_used), _p(r_st), lay.n, _p(scratch), scratch.numel(), _stream())
    assert rc == 0, _lib.status_name(rc)
    return _host(r_len, r_used, r_st, d_out)


def run_lz4(lay, dictionary=None):
    import torch
    from swcompression_b200 import _lib
    d_in, d_off, d_len = _dev(lay.buf), _dev(lay.offs), _dev(lay.lens)
    d_ooff, d_ocap = _dev(lay.out_off), _dev(lay.out_cap)
    d_out = torch.full((lay.total,), H.SENTINEL, dtype=torch.uint8, device="cuda")
    r_len, r_used, r_st = _results(lay.n)
    d_dict, p_dict = None, None
    if dictionary is not None:           # the dictionary at an odd address between non-zero bytes
        d_dict = _dev(np.frombuffer(b"\xFF" * 13 + dictionary + b"\xFF" * 64, dtype=np.uint8).copy())
        p_dict = C.c_void_p(d_dict.data_ptr() + 13)
    rc = _lib.lib().swc_lz4_block_decompress_batch(_p(d_in), _p(d_off), _p(d_len), p_dict, len(dictionary or b""), _p(d_out),
                                                   _p(d_ooff), _p(d_ocap), _p(r_len), _p(r_st), lay.n, _stream())
    assert rc == 0, _lib.status_name(rc)
    return _host(r_len, r_used, r_st, d_out)


def run_bzip2(lay):
    import torch
    from swcompression_b200 import _lib
    d_in, d_off, d_len = _dev(lay.buf), _dev(lay.offs), _dev(lay.lens)
    d_ooff, d_ocap = _dev(lay.out_off), _dev(lay.out_cap)
    d_out = torch.full((lay.total,), H.SENTINEL, dtype=torch.uint8, device="cuda")
    r_len, r_used, r_st = _results(lay.n)
    rc = _lib.lib().swc_bzip2_decompress_batch(_p(d_in), _p(d_off), _p(d_len), _p(d_out), _p(d_ooff), _p(d_ocap),
                                               _p(r_len), _p(r_used), _p(r_st), lay.n, _stream())
    assert rc == 0, _lib.status_name(rc)
    return _host(r_len, r_used, r_st, d_out)


def run_lzma2(lay):
    import torch
    from swcompression_b200 import _lib
    d_in, d_off, d_len = _dev(lay.buf), _dev(lay.offs), _dev(lay.lens)
    d_aux = _dev(np.array([u.aux for u in lay.units], dtype=np.uint8))
    d_ooff, d_ocap = _dev(lay.out_off), _dev(lay.out_cap)
    d_out = torch.full((lay.total,), H.SENTINEL, dtype=torch.uint8, device="cuda")
    r_len, r_used, r_st = _results(lay.n)
    rc = _lib.lib().swc_lzma2_decompress_batch(_p(d_in), _p(d_off), _p(d_len), _p(d_aux), _p(d_out), _p(d_ooff), _p(d_ocap),
                                               _p(r_len), _p(r_used), _p(r_st), lay.n, _stream())
    assert rc == 0, _lib.status_name(rc)
    return _host(r_len, r_used, r_st, d_out)


def run_lzma(lay):
    import torch
    from swcompression_b200 import _lib
    d_in, d_off, d_len = _dev(lay.buf), _dev(lay.offs), _dev(lay.lens)
    d_props = _dev(np.array([u.aux[0] for u in lay.units], dtype=np.uint32))
    d_dsz = _dev(np.array([u.aux[1] for u in lay.units], dtype=np.int64))
    d_usz = _dev(np.array([u.aux[2] for u in lay.units], dtype=np.int64))
    d_ooff, d_ocap = _dev(lay.out_off), _dev(lay.out_cap)
    d_out = torch.full((lay.total,), H.SENTINEL, dtype=torch.uint8, device="cuda")
    r_len, r_used, r_st = _results(lay.n)
    rc = _lib.lib().swc_lzma_decompress_batch(_p(d_in), _p(d_off), _p(d_len), _p(d_props), _p(d_dsz), _p(d_usz), _p(d_out),
                                              _p(d_ooff), _p(d_ocap), _p(r_len), _p(r_used), _p(r_st), lay.n, _stream())
    assert rc == 0, _lib.status_name(rc)
    return _host(r_len, r_used, r_st, d_out)


# ----------------------------------------------------------------------------------------------------------- Deflate
def deflate_small_batches(oracle):
    """Both small hostile Deflate batches (< 20 000 units: the warp-per-unit decoder unless SWC_DEFLATE_K1 forces another),
    without and with start bits; over-subscribed code sets among them take the slow kernel."""
    _, make = H.LAYOUT_SETS["deflate"]
    lay = Layout("deflate", oracle, make(), 201)
    lay.check(*run_both(lay, run_deflate))
    lay.check(*run_both(lay, run_deflate, start_bits=np.zeros(lay.n, dtype=np.uint8)))
    _, make = H.LAYOUT_SETS["deflate_shifted"]
    lay = Layout("deflate", oracle, make(), 202)
    lay.check(*run_both(lay, run_deflate, start_bits=[u.aux for u in lay.units]))


def test_deflate_warp_kernel_and_slow_kernel(oracle):
    deflate_small_batches(oracle)


def test_deflate_small_batches_through_lut_kernel():
    """The table-lookup decoder (inflate_lut.cu) on the same small hostile batches: SWC_DEFLATE_K1=lut is read once per
    process, so they run in a child process."""
    env = dict(os.environ, SWC_DEFLATE_K1="lut")
    env["PYTHONPATH"] = os.pathsep.join([ROOT, os.path.join(ROOT, "oracle"), os.path.join(ROOT, "tests")] +
                                        ([env["PYTHONPATH"]] if env.get("PYTHONPATH") else []))
    flags = ["-s"] if sys.flags.no_user_site else []
    code = "import swco, test_gpu_layout as T; T.deflate_small_batches(swco)"
    p = subprocess.run([sys.executable] + flags + ["-c", code], cwd=ROOT, env=env, stdout=subprocess.PIPE,
                       stderr=subprocess.PIPE, text=True, timeout=600)
    assert p.returncode == 0, p.stderr[-4000:]


def test_deflate_lut_kernel_20000_hostile_units(oracle):
    """>= 20 000 units take the benched pair (inflate_lut_kernel + lz_resolve_kernel; the slow kernel for over-subscribed
    sets).  Distinct units are re-packed, not tiled, so each meets many residues and neighbour kinds; with start bits."""
    _, make = H.LAYOUT_SETS["deflate_large"]
    distinct = make()
    units = [distinct[j % len(distinct)] for j in range(20480)]
    lay = Layout("deflate", oracle, units, 203)
    lay.check(*run_both(lay, run_deflate, start_bits=[u.aux for u in units]))


def test_deflate_host_batch(oracle):
    """swc_deflate_decompress_batch_host at n < 4096 (one slice) and n >= 4096 (slices over three streams): unaligned units
    between foreign bytes, and the caller's bytes between and around the output regions stay as they were."""
    from swcompression_b200 import _lib
    _, make = H.LAYOUT_SETS["deflate"]
    distinct = [u for u in make() if u.aux == 0]
    for n in (len(distinct), 4500):
        lay = Layout("deflate", oracle, [distinct[j % len(distinct)] for j in range(n)], 204 + n)
        out = np.full(lay.total, H.SENTINEL, dtype=np.uint8)
        r_len, r_used, r_st = np.zeros(n, dtype=np.uint64), np.zeros(n, dtype=np.uint64), np.full(n, -1, dtype=np.int32)
        vp = lambda a: a.ctypes.data_as(C.c_void_p)
        rc = _lib.lib().swc_deflate_decompress_batch_host(vp(lay.buf), vp(lay.offs), vp(lay.lens), len(lay.buf), vp(out),
                                                          vp(lay.out_off), vp(lay.out_cap), lay.total, vp(r_len), vp(r_used),
                                                          vp(r_st), n)
        assert rc == 0, _lib.status_name(rc)
        lay.check(r_st, r_len, r_used, out)


# ----------------------------------------------------------------------------------------------------------- LZ4
def test_lz4_parse_and_exec_kernels(oracle):
    _, make = H.LAYOUT_SETS["lz4_block"]
    lay = Layout("lz4_block", oracle, make(), 205)
    lay.check(*run_both(lay, run_lz4), consumed=False)


def test_lz4_host_batch(oracle):
    """swc_lz4_block_decompress_batch_host leaves the caller's bytes between and around the output regions alone."""
    from swcompression_b200 import _lib
    _, make = H.LAYOUT_SETS["lz4_block"]
    lay = Layout("lz4_block", oracle, make(), 214)
    out = np.full(lay.total, H.SENTINEL, dtype=np.uint8)
    r_len, r_st = np.zeros(lay.n, dtype=np.uint64), np.full(lay.n, -1, dtype=np.int32)
    vp = lambda a: a.ctypes.data_as(C.c_void_p)
    rc = _lib.lib().swc_lz4_block_decompress_batch_host(vp(lay.buf), vp(lay.offs), vp(lay.lens), len(lay.buf), vp(out),
                                                        vp(lay.out_off), vp(lay.out_cap), lay.total, vp(r_len), vp(r_st), lay.n)
    assert rc == 0, _lib.status_name(rc)
    lay.check(r_st, r_len, None, out, consumed=False)


def test_lz4_fallback_kernel_literal_run_over_16_mib(oracle):
    """Literal runs of >= 2^24 bytes do not fit the parse kernel's records: such a block (as the last run, and followed by a
    match) goes to lz4_fallback_kernel in the same batch as ordinary blocks, at a 16-byte-congruent and an odd residue."""
    rng = random.Random(206)
    big = np.random.Generator(np.random.PCG64(206)).integers(0, 256, (1 << 24) + 4096, dtype=np.uint8).tobytes()
    tail_run = big + bytes(1000) + big[:40]
    units = [H.LayoutUnit(H.lz4_block_compress(big), raw=big), H.LayoutUnit(H.lz4_block_compress(tail_run), raw=tail_run)]
    units += H.layout_lz4(rng, 8)
    # literal source = unit start + 1 token byte + 65 795 length bytes: residue 13 puts it on a 16-byte boundary
    residues = [13, 7] + [None] * (len(units) - 2)
    lay = Layout("lz4_block", oracle, units, 207, residues=residues)
    assert all(e[0] == 0 for e in lay.expect[:2])
    lay.check(*run_both(lay, run_lz4), consumed=False)


def test_lz4_dictionary_batch(oracle):
    """The dictionary form of swc_lz4_block_decompress_batch: matches reaching into the dictionary, short and long, one
    starting at its first byte and one a byte before it."""
    rng = random.Random(208)
    dict_units = H.lz4_dictionary_units(rng, 24, H.LZ4_DICTIONARY)
    units = dict_units + H.layout_lz4(rng, 6)
    lay = Layout("lz4_block", oracle, units, 209, dictionary=H.LZ4_DICTIONARY)
    k = len(dict_units)
    assert lay.expect[k - 2][0] == 0 and lay.expect[k - 1][0] != 0
    lay.check(*run_both(lay, run_lz4, H.LZ4_DICTIONARY), consumed=False)


# ----------------------------------------------------------------------------------------------------------- BZip2 / LZMA
def test_bzip2_stream_kernel(oracle):
    _, make = H.LAYOUT_SETS["bzip2"]
    lay = Layout("bzip2", oracle, make(), 210)
    lay.check(*run_both(lay, run_bzip2))


def test_lzma2_kernel(oracle):
    _, make = H.LAYOUT_SETS["lzma2"]
    lay = Layout("lzma2", oracle, make(), 211)
    lay.check(*run_both(lay, run_lzma2))


def test_lzma_raw_kernel(oracle):
    _, make = H.LAYOUT_SETS["lzma"]
    lay = Layout("lzma", oracle, make(), 212)
    lay.check(*run_both(lay, run_lzma))


# ----------------------------------------------------------------------------------------------------------- checks
def test_checksum_batches_every_residue(oracle):
    """swc_crc32_batch / swc_xxh32_batch over lengths 0..64 and around 64 KiB at every residue, between non-zero bytes."""
    import torch
    from swcompression_b200 import _lib
    rng = random.Random(213)
    lens = list(range(65)) * 2 + [65535, 65536, 65537, 65551] * 4
    units = [H.random_bytes(rng, k) for k in lens]
    buf, offs, ln = H.pack_hostile(units, rng)
    assert set((offs % 16).tolist()) == set(range(16))
    d_in, d_off, d_len = _dev(buf), _dev(offs), _dev(ln)
    n = len(units)
    d_crc = torch.full((n,), 0x0BADF00D, dtype=torch.int32, device="cuda")
    d_crc0 = torch.full((n,), 0x0BADF00D, dtype=torch.int32, device="cuda")
    d_xxh = torch.zeros(n, dtype=torch.int32, device="cuda")
    d_st = _dev(np.zeros(n, dtype=np.int32))
    L = _lib.lib()
    assert L.swc_crc32_batch(_p(d_in), _p(d_off), _p(d_len), None, _p(d_crc), n, _stream()) == 0
    assert L.swc_crc32_batch(_p(d_in), _p(d_off), _p(d_len), _p(d_st), _p(d_crc0), n, _stream()) == 0
    assert L.swc_xxh32_batch(_p(d_in), _p(d_off), _p(d_len), _p(d_xxh), n, _stream()) == 0
    torch.cuda.synchronize()
    crc, crc0 = d_crc.cpu().numpy().view(np.uint32), d_crc0.cpu().numpy().view(np.uint32)
    xxh = d_xxh.cpu().numpy().view(np.uint32)
    bad = [(i, len(u), int(offs[i]) % 16) for i, u in enumerate(units)
           if not (crc[i] == crc0[i] == zlib.crc32(u) and xxh[i] == oracle.xxh32(u))]
    assert not bad, f"{len(bad)} of {n} checksums differ (index, length, residue): {bad[:8]}"
