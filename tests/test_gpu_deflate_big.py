"""Deflate units that decode to 2 GiB and more (tests/deflate_big_cases.py) through swc_deflate_decompress_batch, up to
the largest output a unit may have (OUT_MAX = 0xFFFFFFF0 bytes) and just past it.

Every batch puts its output base 4 GiB into a sentinel-filled buffer the test owns, so that a store whose 32-bit position
went negative (4 GiB early) lands in memory the test checks.  Each big unit sits between sentinel gaps with a small
neighbour unit behind it that must decode exactly; the same streams also run at capacity 0, where they must report
OUTPUT_OVERFLOW with their exact size.  Outputs are compared with the pattern on the device, in slices.

- K1w (inflate_warp_kernel) takes these small batches by default; K1L (inflate_lut_kernel) runs them in a child process
  with SWC_DEFLATE_K1=lut;
- the 2^31 + 1 and ceiling cases at all 16 output phases (offset mod 16), every other size at one phase each;
- the units past the ceiling at capacity 0 and at capacity OUT_MAX: SWC_ERR_UNSUPPORTED, nothing written;
- Deflate.decompress, GzipArchive.unarchive and ZlibArchive.unarchive on a 3 GiB stream.

Batches take as many big units as the free device memory allows (each needs its output and 4/3 of it in record
scratch); a device with less than about 17 GB free skips."""
import os
import struct
import subprocess
import sys
import zlib

import numpy as np
import pytest

import deflate_big_cases as B
import helpers as H
from test_gpu_layout import _dev, _p, _stream

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
OK, OVERFLOW, UNSUPPORTED = 0, 1, 6
MARGIN = 1 << 32                # sentinel bytes in front of the output base
GAP = 4096                      # sentinel bytes around every region
SLICE = 256 << 20
NEIGHBOUR = H.textlike(5000, 41)
NEIGHBOUR_Z = H.raw_deflate(NEIGHBOUR)
MAX_GROUP = 4                   # big units per batch at most


def _unit_bytes(cap):
    return cap + cap * 4 // 3 + 2 * GAP


def _device_room():
    import torch
    torch.cuda.empty_cache()                    # what earlier batches left in the caching allocator
    free, _ = torch.cuda.mem_get_info()
    return free - MARGIN - (3 << 30)            # the margin, the pattern tensors and comparison temporaries


def _need_device(cap):
    room = _device_room()
    if room < _unit_bytes(cap):
        pytest.skip(f"{(room + MARGIN + (3 << 30)) >> 20} MiB free on the device; a unit of {cap >> 20} MiB needs about "
                    f"{(_unit_bytes(cap) + MARGIN + (3 << 30)) >> 20} MiB")


def _groups(items):
    """items (case, phase, cap) -> lists that fit the free device memory together, in order"""
    room = _device_room()
    out, cur, used = [], [], 0
    for it in items:
        need = _unit_bytes(it[2])
        if cur and (used + need > room or len(cur) == MAX_GROUP):
            out.append(cur)
            cur, used = [], 0
        assert need <= room, f"{need >> 20} MiB needed for one unit, {room >> 20} MiB available"
        cur.append(it)
        used += need
    return out + ([cur] if cur else [])


def _tiled(torch):
    reps = (SLICE + 2 * B.P) // B.P + 1
    return torch.tensor(np.frombuffer(B.SEED * reps, dtype=np.uint8), device="cuda")


def run_group(items):
    """one batch: for every (case, phase, cap) a region of `cap` bytes at that phase followed by the small neighbour, each
    behind GAP sentinel bytes, then every case once more at capacity 0.  Checks statuses, sizes, consumed bits, the
    pattern, the neighbours and every byte outside the written regions; -> list of what differs"""
    import torch
    from swcompression_b200 import _lib
    L = _lib.lib()
    units, regions = [], []     # units: (data, out_off, cap, expected status, expected len, nbits); regions: (off, len)
    pos = 0
    for c, phase, cap in items:
        pos = (pos + GAP + 15) // 16 * 16 + phase
        units.append((c.data, pos, cap, OK if c.decodes and cap >= c.size else UNSUPPORTED if not c.decodes else OVERFLOW,
                      c.size if c.decodes else None, c.nbits if c.decodes else None))
        if c.decodes and cap >= c.size:
            regions.append((pos, c.size, c))
        pos += cap
        pos += GAP + 7
        units.append((NEIGHBOUR_Z, pos, len(NEIGHBOUR), OK, len(NEIGHBOUR), None))
        regions.append((pos, len(NEIGHBOUR), None))
        pos += len(NEIGHBOUR)
    for c, _, _ in items:
        pos += 16
        units.append((c.data, pos, 0, OVERFLOW if c.decodes else UNSUPPORTED, c.size if c.decodes else None,
                      c.nbits if c.decodes else None))
    total = pos + GAP
    n = len(units)
    buf, offs, lens, p = [], [], [], 0
    for d, *_ in units:                         # inputs at odd offsets between junk bytes
        buf.append(b"\x5A" * 3)
        p += 3
        offs.append(p)
        lens.append(len(d))
        buf.append(d)
        p += len(d)
    buf.append(b"\x5A" * 64)
    d_in = _dev(np.frombuffer(b"".join(buf), dtype=np.uint8).copy())
    d_off, d_len = _dev(np.array(offs, dtype=np.uint64)), _dev(np.array(lens, dtype=np.uint64))
    d_ooff = _dev(np.array([u[1] for u in units], dtype=np.uint64))
    d_ocap = _dev(np.array([u[2] for u in units], dtype=np.uint64))
    d_buf = torch.full((MARGIN + total,), H.SENTINEL, dtype=torch.uint8, device="cuda")
    r_len = torch.zeros(n, dtype=torch.int64, device="cuda")
    r_used = torch.zeros(n, dtype=torch.int64, device="cuda")
    r_st = torch.full((n,), -1, dtype=torch.int32, device="cuda")
    scratch = torch.empty(L.swc_deflate_batch_scratch_bytes(n, total), dtype=torch.uint8, device="cuda")
    import ctypes as C
    out_base = C.c_void_p(d_buf.data_ptr() + MARGIN)
    rc = L.swc_deflate_decompress_batch(_p(d_in), _p(d_off), _p(d_len), None, out_base, _p(d_ooff), _p(d_ocap), total,
                                        _p(r_len), _p(r_used), _p(r_st), n, _p(scratch), scratch.numel(), _stream())
    assert rc == 0, _lib.status_name(rc)
    torch.cuda.synchronize()
    del scratch
    st, ln, used = r_st.cpu().tolist(), r_len.cpu().tolist(), r_used.cpu().tolist()
    bad = []
    names = []
    for c, phase, cap in items:
        names += [f"{c.name}@{phase}/cap {cap:#x}", f"neighbour of {c.name}@{phase}"]
    names += [f"{c.name}/cap 0" for c, _, _ in items]
    for i, (u, name) in enumerate(zip(units, names)):
        want = (u[3], u[4], u[5])
        got = (st[i], ln[i] if u[4] is not None else None, used[i] if u[5] is not None else None)
        if got != want:
            bad.append((name, "status, out_len, consumed", got, want))
    tiled = _tiled(torch)
    out = d_buf[MARGIN:]
    want_nb = torch.tensor(np.frombuffer(NEIGHBOUR, dtype=np.uint8), device="cuda")
    for off, size, c in regions:
        if c is None:
            if not torch.equal(out[off:off + size], want_nb):
                bad.append(("neighbour", off, "wrong bytes"))
            continue
        for a in range(0, size, SLICE):
            b = min(a + SLICE, size)
            k = a % B.P
            got = out[off + a:off + b]
            if not torch.equal(got, tiled[k:k + b - a]):
                first = int(torch.nonzero(got != tiled[k:k + b - a])[0].item())
                bad.append((c.name, off % 16, f"byte {a + first:#x} of {size:#x} differs"))
                break
    # everything else is sentinel: the margin and every gap
    def fence(t, what):
        for a in range(0, t.numel(), SLICE):
            s = t[a:a + SLICE]
            if not bool((s == H.SENTINEL).all()):
                first = int(torch.nonzero(s != H.SENTINEL)[0].item())
                bad.append((what, f"byte {a + first:#x} changed"))
                return
    fence(d_buf[:MARGIN], "the 4 GiB in front of the output base")
    edges = sorted((off, off + size) for off, size, _ in regions)
    prev = 0
    for a, b in edges + [(total, total)]:
        fence(out[prev:a], f"gap before output byte {a:#x}")
        prev = b
    return bad


def _run(items):
    import torch
    bad = []
    for g in _groups(items):
        bad += run_group(g)
        torch.cuda.empty_cache()
    assert not bad, f"{len(bad)} differences: {bad[:10]}"


def phase_items():
    cases = [B.crossing(), B.ceiling()]
    return [(c, ph, c.size) for c in cases for ph in range(16)]


def length_items():
    return [(c, (5 * i + 3) % 16, c.size) for i, c in enumerate(B.lengths())]


def past_items():
    return [(c, (3 * i + 1) % 16, B.OUT_MAX) for i, c in enumerate(B.past_ceiling())]


def phases():
    _run(phase_items())


def lengths():
    _run(length_items())


def past_ceiling():
    _run(past_items())


def _child(kernel, fn):
    env = dict(os.environ, SWC_DEFLATE_K1=kernel)
    env["PYTHONPATH"] = os.pathsep.join([ROOT, os.path.join(ROOT, "oracle"), os.path.join(ROOT, "tests")] +
                                        ([env["PYTHONPATH"]] if env.get("PYTHONPATH") else []))
    flags = ["-s"] if sys.flags.no_user_site else []
    code = f"import test_gpu_deflate_big as T; T.{fn}()"
    p = subprocess.run([sys.executable] + flags + ["-c", code], cwd=ROOT, env=env, stdout=subprocess.PIPE,
                       stderr=subprocess.PIPE, text=True, timeout=1800)
    assert p.returncode == 0, p.stderr[-4000:]


def test_phases_warp_kernel():
    """2^31 + 1 and OUT_MAX bytes, both ending on a match, at every output phase"""
    _need_device(B.OUT_MAX)
    phases()


def test_phases_lut_kernel():
    _need_device(B.OUT_MAX)
    _child("lut", "phases")


def test_lengths_warp_kernel():
    """2^31 - 1, 2^31, 2^31 + 1, 3 GiB and OUT_MAX - k, ending on matches, literal runs and stored blocks"""
    _need_device(B.OUT_MAX)
    lengths()


def test_lengths_lut_kernel():
    _need_device(B.OUT_MAX)
    _child("lut", "lengths")


def test_past_ceiling_warp_kernel():
    """one byte past OUT_MAX by a match and by a literal, 2^32 by sixteen literals, a stored block across both: each
    SWC_ERR_UNSUPPORTED at capacity OUT_MAX and at capacity 0, and no byte written"""
    _need_device(B.OUT_MAX)
    past_ceiling()


def test_past_ceiling_lut_kernel():
    _need_device(B.OUT_MAX)
    _child("lut", "past_ceiling")


# ------------------------------------------------------------------------------------------------ single calls
def test_single_calls_3_gib():
    """Deflate.decompress, GzipArchive.unarchive and ZlibArchive.unarchive of a 3 GiB stream: the first attempt
    overflows its guess, the exact-size retry decodes it; CRC-32 and Adler-32 from zlib, bytes compared in slices"""
    import torch
    import swcompression_b200 as S
    from swcompression_b200 import _lib
    size = 3 << 30
    _need_device(size)
    with open("/proc/meminfo") as f:
        avail = next(int(l.split()[1]) << 10 for l in f if l.startswith("MemAvailable:"))
    if avail < 8 << 30:
        pytest.skip(f"{avail >> 20} MiB of host memory available; the call needs about 8 GiB")
    c = B.build(size, "stored", name="3GiB-stored")
    step = 64 << 20
    crc, adler = 0, 1
    for a in range(0, size, step):
        piece = B.expected(a, min(step, size - a)).tobytes()
        crc, adler = zlib.crc32(piece, crc), zlib.adler32(piece, adler)
    gz = b"\x1f\x8b\x08\x00\x00\x00\x00\x00\x00\xff" + c.data + struct.pack("<II", crc, size & 0xFFFFFFFF)
    zl = b"\x78\x01" + c.data + struct.pack(">I", adler)
    bad = []
    try:
        for name, fn, arg in (("Deflate.decompress", S.Deflate.decompress, c.data),
                              ("GzipArchive.unarchive", S.GzipArchive.unarchive, gz),
                              ("ZlibArchive.unarchive", S.ZlibArchive.unarchive, zl)):
            out = fn(arg)
            if len(out) != size:
                bad.append((name, len(out)))
            else:
                a = np.frombuffer(out, dtype=np.uint8)
                for p in range(0, size, step):
                    if not np.array_equal(a[p:p + step], B.expected(p, min(step, size - p))):
                        bad.append((name, f"slice at {p:#x}"))
                        break
            del out
    finally:
        _lib.lib().swc_release_scratch()
        torch.cuda.empty_cache()
    assert not bad, bad
