"""Block headers on the generic Deflate decoder (inflate_slow_kernel).  The batch decoders hand a unit to that kernel
when one of its code sets is over-subscribed, so its header parse otherwise meets only valid headers and truncated ones.
Here every case of families 2 and 5 of tests/deflate_cases.py (header edges, stored blocks, with all their header
errors: HLIT 287 / 288, 16 first, repeats past the count, LEN / NLEN, ...) is put behind a non-final dynamic block with an
over-subscribed lit/len set, which sends the whole unit to inflate_slow_kernel.  The cases run as a batch on the default
path (K1w), in a child process with SWC_DEFLATE_K1=lut (K1L), and through Deflate.decompress_from; the status, and for
valid streams the bytes and consumed bits, must equal the oracle's."""
import random

import pytest

import deflate_cases as D
from deflate_writer import DeflateWriter, Match
from test_gpu_deflate_handmade import _child, case_batches

pytestmark = pytest.mark.gpu


class SlowCase:
    __slots__ = ("name", "data", "start_bit", "nbits", "expect", "status")

    def __init__(self, name, data, nbits, expect, status):
        self.name, self.data, self.start_bit, self.nbits, self.expect, self.status = name, data, 0, nbits, expect, status


def _prefix():
    """an over-subscribed dynamic block and an empty stored block that ends it on a byte boundary -> (bytes, output)"""
    rng = random.Random(2501)
    w = DeflateWriter(oversub="lit")
    w.dynamic([bytes(rng.randrange(97, 123) for _ in range(40)), Match(5, 3)])
    w.oversub = None
    w.stored(b"")
    data, end = w.finish()
    assert w.trace.blocks[0][4] == ("lit",) and end == 8 * len(data)
    return data, bytes(w.out)


def slow_cases():
    pre, out = _prefix()
    cases = []
    for c in list(D.family2()) + list(D.family5()):
        assert c.start_bit == 0
        cases.append(SlowCase(c.name + "/behind_oversub", pre + c.data, 8 * len(pre) + c.nbits,
                              None if c.expect is None else out + c.expect, c.status))
    assert sum(c.expect is None for c in cases) >= 15
    return cases


def slow_batches(oracle):
    case_batches(oracle, slow_cases())


def test_headers_slow_kernel_from_warp_kernel(oracle):
    slow_batches(oracle)


def test_headers_slow_kernel_from_lut_kernel():
    _child("lut", "slow_batches", module="test_gpu_deflate_headers")


def test_headers_slow_kernel_single_stream():
    import swcompression_b200 as S
    bad = []
    for c in slow_cases():
        try:
            out, used = S.Deflate.decompress_from(c.data, c.start_bit)
            got = (0, out, used)
        except S.SWCompressionError as e:
            got = (e.code, None, None)
        if got != ((0, c.expect, c.nbits) if c.expect is not None else (c.status, None, None)):
            bad.append((c.name, got[0], c.status, got[2], c.nbits))
    assert not bad, f"{len(bad)} cases differ: {bad[:8]}"
