"""The hand-built ZIP catalogue (zip_cases.py) through swc_zip_open / swc_zip_info against the oracle: status, entries and
the wrongCRC payload; byte truncations of the small containers; the whole catalogue again with the entry data at every
residue mod 16; and containers large enough to take the batch paths a handful of entries never reach — 20 000 Deflate
entries (the table-lookup Huffman kernel, each unit's input running to the end of the container), 70 000 entries (the
Zip64 end record), and 20 000 Deflate entries in front of a stored entry that puts the container past 256 MiB."""
import struct
import zlib

import pytest

import zip_cases as Z
from zip_writer import Entry, build

pytestmark = pytest.mark.gpu


def engine_open(blob):
    """-> (status, [entry dicts]) in the oracle's shape, from ZipContainer.open (the wrongCRC payload on 910)"""
    import swcompression_b200 as S
    try:
        got, st = S.ZipContainer.open(blob), 0
    except S.SWCompressionError as e:
        got, st = e.payload or [], e.code
    return st, [(g.info.name, g.data, g.info.crc, g.info.size, g.info.type == "directory") for g in got]


def engine_info(blob):
    import swcompression_b200 as S
    try:
        return 0, [(i.name, i.size, i.crc, i.type == "directory") for i in S.ZipContainer.info(blob)]
    except S.SWCompressionError as e:
        return e.code, []


def oracle_view(oracle, blob):
    from swcompression_b200.api import _zip_text
    st, ents = oracle.zip_open(blob, max_entries=1 << 17)
    ist, ients = oracle.zip_open(blob, info_only=True, max_entries=1 << 17)
    opened = [(_zip_text(e["name"], e["utf8"]), e["data"], e["crc"], e["size"], e["is_directory"]) for e in ents]
    listed = [(_zip_text(e["name"], e["utf8"]), e["size"], e["crc"], e["is_directory"]) for e in ients]
    return (st, opened), (ist, listed)


def check(oracle, blob, engine_status=None, what=""):
    want_open, want_info = oracle_view(oracle, blob)
    got = engine_open(blob)
    if engine_status is not None:
        assert got[0] == engine_status, what
    else:
        assert got[0] == want_open[0], (what, got[0], want_open[0])
        if got[0] in (0, Z.CRC):
            assert got[1] == want_open[1], what
    assert engine_info(blob) == want_info, what


@pytest.mark.parametrize("c", Z.cases(), ids=lambda c: c.name)
def test_case_matches_oracle(oracle, c):
    assert oracle.zip_open(c.blob)[0] == c.status
    check(oracle, c.blob, c.engine, c.name)


def truncation_points(n):
    """every cut of a container under 160 bytes; of one under 2 KiB, 24 cuts spread over it and every cut of its last 32
    bytes (where the end record, and with it most of the walk, survives)"""
    if n < 160:
        return range(n)
    return sorted(set(range(0, n, max(1, n // 24))) | set(range(n - 32, n)))


def test_truncations_of_small_cases_match_oracle(oracle):
    n = 0
    for c in Z.cases():
        if len(c.blob) > 2048 or c.engine is not None:
            continue
        ks = truncation_points(len(c.blob))
        for k in ks:
            check(oracle, c.blob[:k], what=(c.name, k))
            n += 1
    assert n > 10000


def test_every_residue_mod_16_matches_oracle(oracle):
    for shift in range(1, 16):
        for c in Z.cases(shift):
            assert oracle.zip_open(c.blob)[0] == c.status, (c.name, shift)
            check(oracle, c.blob, c.engine, (c.name, shift))


# ---------------------------------------------------------------------------------------------------------------- scale
def _deflated(i):
    data = b"entry %d: " % i + Z.text(200 + i % 300, i)
    co = zlib.compressobj(6, zlib.DEFLATED, -15)
    return data, co.compress(data) + co.flush()


def _launches(blob):
    import swcompression_b200 as S
    from swcompression_b200 import _lib
    S.ZipContainer.open(build([Entry("w", b"warm")]).blob)                 # module load, arenas
    before = _lib.lib().swc_kernel_launches()
    got = S.ZipContainer.open(blob)
    return got, _lib.lib().swc_kernel_launches() - before


def test_20000_deflate_entries_one_batch():
    ents = []
    for i in range(20000):
        data, p = _deflated(i)
        ents.append(Entry(f"d/{i}", data, p, 8))
    got, launches = _launches(build(ents).blob)
    assert [g.data for g in got] == [e.data for e in ents]
    assert launches < 40, launches


def test_70000_entries_need_the_zip64_end_record():
    ents = [Entry(f"s{i}", b"%d" % i) for i in range(70000)]
    b = build(ents, zip64=True, saturate=("here", "total"))
    assert struct.unpack_from("<H", b.blob, b.eocd_off + 10)[0] == 0xFFFF
    got, launches = _launches(b.blob)
    assert [g.data for g in got] == [e.data for e in ents]
    assert launches < 40, launches


def test_deflate_entries_in_front_of_256_mib_stay_in_the_batch():
    """every Deflate unit's input would run past 2^28 bytes to the end of the container; the entries must still be
    decoded in the batch, not one by one"""
    ents = []
    for i in range(20000):
        data, p = _deflated(i)
        ents.append(Entry(f"d/{i}", data, p, 8))
    big = bytes(range(256)) * ((260 << 20) // 256)
    ents.append(Entry("big.bin", big))
    blob = build(ents).blob
    assert len(blob) > 1 << 28
    got, launches = _launches(blob)
    print(f"launches: {launches}")
    assert len(got) == len(ents)
    assert all(g.data == e.data for g, e in zip(got, ents))
    assert launches < 40, launches
