"""The single-archive calls swc_gzip_unarchive (with consumed_bytes) and swc_zlib_unarchive against the oracle's gzip_unarchive /
zlib_unarchive: status, output bytes on OK and on the payload-carrying statuses, and consumed bytes, on the catalogue of
tests/unarchive_cases.py, the Deflate catalogue inside members, truncations, an output far past the first size guess, and
stored members around the 4 KiB checksum chunk with an intact and a flipped CRC-32 / Adler-32."""
import ctypes as C
import random

import numpy as np
import pytest

import helpers as H
import unarchive_cases as U
from test_gpu_unarchive_batch import _truncations

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def S():
    import torch
    assert torch.cuda.is_available()
    import swcompression_b200 as S
    return S


def _single(fmt, data):
    """(status, output, consumed bytes) of one call; zlib's single call reports no consumed count"""
    from swcompression_b200 import _lib
    L = _lib.lib()
    buf, n = _lib.inbuf(data)
    out, ol, used = C.c_void_p(), C.c_size_t(), C.c_size_t(12345)
    if fmt == "gzip":
        st = L.swc_gzip_unarchive(buf, n, C.byref(out), C.byref(ol), C.byref(used))
    else:
        st = L.swc_zlib_unarchive(buf, n, C.byref(out), C.byref(ol))
    return st, _lib.take(out, ol), used.value if fmt == "gzip" else None


def _differences(oracle, arcs):
    bad = []
    for fmt, name, data in arcs:
        ost, oout, oused = U.oracle_unarchive(oracle, fmt, data)
        st, out, used = _single(fmt, data)
        carries = ost in (U.OK,) + U.PAYLOAD_CARRYING
        if st != ost:
            bad.append((name, "status", st, ost))
        elif carries and out != oout:
            bad.append((name, "payload", len(out), len(oout)))
        elif not carries and out != b"":
            bad.append((name, "output of a failed call", len(out)))
        elif used is not None and used != oused:
            bad.append((name, "consumed", used, oused))
    return bad


def test_catalogue(S, oracle):
    """every archive of unarchive_cases: headers, trailers, the Deflate catalogue wrapped, Python's gzip / zlib at every level"""
    arcs = [(a.fmt, a.name, a.data) for a in U.cases()]
    bad = _differences(oracle, arcs)
    assert not bad, f"{len(bad)} of {len(arcs)} differ: {bad[:8]}"


def test_deflate_member_cases(S, oracle):
    """the Deflate catalogue's bit-0 streams inside members, and damaged dynamic headers the slow kernel takes"""
    arcs = [(a.fmt, a.name, a.data) for a in U.deflate_member_cases()]
    for j, u in enumerate(H.layout_malformed_deflate(random.Random(71), 80)):
        arcs.append(("gzip", f"gzip malformed {j}", U.GZIP_HEAD + u.data + bytes(8)))
        arcs.append(("zlib", f"zlib malformed {j}", U.ZLIB_HEAD + u.data + bytes(4)))
    bad = _differences(oracle, arcs)
    assert not bad, f"{len(bad)} of {len(arcs)} differ: {bad[:8]}"


def test_truncations(S, oracle):
    """every cut of small archives and random cuts of large ones"""
    arcs = [("gzip" if a[:2] == b"\x1f\x8b" else "zlib", f"cut {len(a)} at {k}", a[:k]) for a, k in _truncations(random.Random(60))]
    bad = _differences(oracle, arcs)
    assert not bad, f"{len(bad)} of {len(arcs)} differ: {bad[:8]}"


def test_output_past_the_first_guess(S, oracle):
    """members that expand far beyond 4 x their input + 64 KiB: the first attempt overflows and the rerun at the exact size
    decodes, with the same consumed bytes"""
    raws = [bytes(8 << 20), H.textlike(1 << 14, 90) * 512]
    arcs = []
    for j, raw in enumerate(raws):
        g, z = U.gzip_member(raw, 9), U.zlib_stream(raw, 9)
        assert 4 * len(g) + 65536 < len(raw)
        arcs += [("gzip", f"gzip {j}", g), ("zlib", f"zlib {j}", z), ("gzip", f"gzip {j} + rest", g + g[:30])]
    bad = _differences(oracle, arcs)
    assert not bad, bad


STORED_SIZES = (0, 1, 4095, 4096, 4097, 3 * 4096 + 5, (1 << 20) - 1, (1 << 20) + 1)


def test_checksum_edges(S, oracle):
    """stored members (Deflate is a copy) at and around multiples of the 4 KiB checksum chunk, each intact and with the
    CRC-32 / Adler-32 flipped in its first and in its last byte"""
    arcs = []
    for n in STORED_SIZES:
        raw = np.random.default_rng(n).integers(0, 256, n, dtype=np.uint8).tobytes()
        g, z = U.gzip_member(raw, 0), U.zlib_stream(raw, 0)
        arcs += [("gzip", f"gzip {n}", g), ("zlib", f"zlib {n}", z)]
        for at in (-8, -5):
            b = bytearray(g); b[at] ^= 0x10
            arcs.append(("gzip", f"gzip {n} crc byte {at}", bytes(b)))
        for at in (-4, -1):
            b = bytearray(z); b[at] ^= 0x10
            arcs.append(("zlib", f"zlib {n} adler byte {at}", bytes(b)))
    bad = _differences(oracle, arcs)
    assert not bad, bad
    statuses = [U.oracle_unarchive(oracle, fmt, data)[0] for fmt, _, data in arcs]
    assert [statuses.count(s) for s in (U.OK, U.GZ_CRC, U.ZL_ADLER)] == [2 * len(STORED_SIZES)] * 3
