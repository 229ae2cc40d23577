"""swc_gzip_archive_header and the archive size bounds (swc_gzip_archive_max_bytes, swc_zlib_archive_max_bytes) against
the CPU restatement of GzipArchive.archive and ZlibArchive.archive.  No device: the header builder runs on the host."""
import ctypes as C
import random

import pytest

import archive_options as AO
import deflatec_cases as K
import helpers as H


@pytest.fixture(scope="module")
def oc():
    import swco_deflatec
    swco_deflatec.lib()
    return swco_deflatec


def oracle_header(oc, data, kw):
    st, whole, _ = oc.gzip_archive(data, **kw)
    assert st == 0
    return whole[:len(whole) - len(oc.deflate_compress(data)[1]) - 8]


def test_header_equals_oracle_prefix_over_option_grid(oc):
    from swcompression_b200 import GzipArchive
    grid = AO.grid()
    assert len(grid) == len(AO.COMMENTS) * len(AO.NAMES) * 2 * len(AO.OS_BYTES)
    for api, kw in grid:
        assert GzipArchive.archive_header(**api) == oracle_header(oc, b"x", kw), api


def test_header_of_every_mtime_and_extra_set(oc):
    from swcompression_b200 import GzipArchive
    for mt in AO.MTIMES:
        for ex in AO.extra_sets():
            api = dict(modificationTime=mt, extraFields=ex, writeHeaderCRC=True)
            assert GzipArchive.archive_header(**api) == oracle_header(oc, b"", AO.oracle_keywords(api)), (mt, len(ex))


def test_xlen_65536_is_cannot_encode(oc):
    from swcompression_b200 import ExtraField, GzipArchive
    from swcompression_b200.errors import GzipError
    for ex in ([ExtraField(1, 1, bytes(65532))], [ExtraField(1, 1, bytes(30000)), ExtraField(2, 2, bytes(35528))]):
        with pytest.raises(GzipError) as e:
            GzipArchive.archive_header(extraFields=ex)
        assert e.value.code == 607


def test_short_cap_reports_exact_len():
    from swcompression_b200 import _lib
    from swcompression_b200.api import _gzip_options
    L = _lib.lib()
    o, _keep = _gzip_options(comment="a comment", fileName="f.bin", writeHeaderCRC=True)
    n = C.c_size_t(0)
    assert L.swc_gzip_archive_header(C.byref(o), None, 0, C.byref(n)) == 1
    full = n.value
    assert full == 10 + len("f.bin") + 1 + len("a comment") + 1 + 2
    for cap in (1, full - 1):
        buf = C.create_string_buffer(b"\x5a" * full, full)
        n = C.c_size_t(0)
        assert L.swc_gzip_archive_header(C.byref(o), buf, cap, C.byref(n)) == 1 and n.value == full
        assert buf.raw == b"\x5a" * full                     # nothing written
    buf = C.create_string_buffer(full)
    assert L.swc_gzip_archive_header(C.byref(o), buf, full, C.byref(n)) == 0 and n.value == full
    assert buf.raw[:2] == b"\x1f\x8b"


def bound_units():
    rng = random.Random(5)
    units = [d for _, d in K.cases()]
    for n in (0, 1, 2, 3, 100, 5000, 65535, 65536, 70000, 300000):
        units += [H.random_bytes(rng, n), H.textlike(n, n), bytes(n)]
    return units


def test_max_bytes_cover_oracle_archives(oc):
    from swcompression_b200 import GzipArchive, ZlibArchive, _lib
    L = _lib.lib()
    opts = dict(comment="c", fileName="name", writeHeaderCRC=True, extraFields=AO.extra_sets()[2])
    hl = len(GzipArchive.archive_header(**opts))
    kw = AO.oracle_keywords(opts)
    for u in bound_units():
        z = oc.zlib_archive(u)[1]
        g = oc.gzip_archive(u, **kw)[1]
        assert len(z) <= ZlibArchive.max_archive_size(len(u)) == L.swc_zlib_archive_max_bytes(len(u))
        assert len(g) <= GzipArchive.max_archive_size(len(u), **opts) == L.swc_gzip_archive_max_bytes(len(u), hl)
        assert ZlibArchive.max_archive_size(len(u)) == 2 + (9 * len(u) + 17) // 8 + 4
        assert GzipArchive.max_archive_size(len(u), **opts) == hl + (9 * len(u) + 17) // 8 + 8
