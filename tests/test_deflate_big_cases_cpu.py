"""The Deflate streams of tests/deflate_big_cases.py, decoded by zlib: each is valid Deflate, decodes to the size it
claims and holds the periodic pattern everywhere.  The past-the-ceiling cases are valid too, so the limit the GPU decoders
put on them (SWC_ERR_UNSUPPORTED) is the engine's, not the stream's."""
import os
import zlib
from concurrent.futures import ProcessPoolExecutor

import pytest

import deflate_big_cases as B


def _all():
    return B.lengths() + B.past_ceiling()


def test_layout_of_the_catalogue():
    """the sizes the GPU tests rely on: both sides of 2^31, 3 GiB, OUT_MAX - k for k up to 16, every tail kind, and four
    units past OUT_MAX, two of them reaching 2^32"""
    cases = _all()
    sizes = {c.size for c in cases if c.decodes}
    assert {(1 << 31) - 1, 1 << 31, (1 << 31) + 1, 3 << 30, B.OUT_MAX, B.OUT_MAX - 16} <= sizes
    assert {c.tail for c in cases if c.decodes and c.size >= B.OUT_MAX - 16} == {"match", "literal", "stored"}
    over = [c for c in cases if not c.decodes]
    assert len(over) == 4 and {c.tail for c in over} == {"match", "literal", "stored"}
    assert sum(c.size >= 1 << 32 for c in over) == 2
    assert all(len(c.data) < 32 << 20 for c in cases)
    assert len({c.name for c in cases}) == len(cases)


@pytest.mark.parametrize("size", [6000, 6001, 6002, 6257, 6258, 7777])
@pytest.mark.parametrize("tail,tail_len", [("match", 0), ("literal", 1), ("literal", 16), ("stored", 0), ("stored", 700)])
def test_small_streams_of_the_same_layout(size, tail, tail_len):
    c = B.build(size, tail, tail_len)
    out = zlib.decompress(c.data, -15)
    assert len(out) == size and out == B.expected(0, size).tobytes()


def test_pattern_helper():
    assert B.expected(0, 3 * B.P + 5).tobytes() == (B.SEED * 4)[:3 * B.P + 5]
    assert B.expected(B.P * 7 + 9, 300).tobytes() == (B.SEED * 3)[9:309]


def test_every_case_is_valid_deflate():
    """zlib decodes every case, in 64 MiB slices, to exactly its size and the pattern, with nothing after the final
    block (about 6 s of zlib per 4 GiB; the cases run in parallel)"""
    cases = _all()
    workers = max(1, min(len(cases), os.cpu_count() or 1, 8))
    with ProcessPoolExecutor(workers) as ex:
        res = list(ex.map(B.zlib_check, [c.size for c in cases], [c.tail for c in cases], [c.tail_len for c in cases]))
    bad = [(c.name, r) for c, r in zip(cases, res) if r != (c.size, True, None)]
    assert not bad, bad
