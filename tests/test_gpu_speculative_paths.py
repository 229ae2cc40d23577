"""The speculative multi-unit paths are taken on valid archives.

GzipArchive.multiUnarchive, BZip2.multiDecompress and XZArchive.splitUnarchive first decode every unit they can find as
one batch and fall back to the sequential walk on anything that does not validate.  The fallback gives the same bytes,
so the output alone cannot tell whether the batch ran.  The kernel-launch count can: the batch costs a constant number
of launches, the sequential walk at least one per unit."""
import bz2
import gzip
import lzma
import random

import pytest

import helpers as H

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def gpu():
    import torch
    assert torch.cuda.is_available()
    import swcompression_b200 as S
    return S


def _launches(fn, data):
    from swcompression_b200 import _lib
    before = _lib.lib().swc_kernel_launches()
    out = fn(data)
    return out, _lib.lib().swc_kernel_launches() - before


def test_gzip_multi_unarchive_decodes_members_as_one_batch(gpu, oracle):
    rng = random.Random(31)
    raws = [H.textlike(rng.randrange(1, 40000), 300 + i) if i % 9 else b"" for i in range(60)]
    data = b"".join(gzip.compress(r, rng.choice((1, 6, 9))) for r in raws)
    ost, oparts, _ = oracle.gzip_multi_unarchive(data)
    assert ost == 0 and oparts == raws
    members, launches = _launches(gpu.GzipArchive.multiUnarchive, data)
    assert [m.data for m in members] == oparts
    assert launches < len(raws), launches


def test_bzip2_multi_decompress_decodes_streams_as_one_batch(gpu, oracle):
    rng = random.Random(32)
    raws = [H.textlike(rng.choice([70, 500, 3000, 40000]), 400 + i) if i % 7 else b"" for i in range(40)]
    data = b"".join(bz2.compress(r, rng.choice([1, 9])) for r in raws)
    ost, oparts, _ = oracle.bzip2_multi_decompress(data)
    assert ost == 0 and oparts == raws
    parts, launches = _launches(gpu.BZip2.multiDecompress, data)
    assert parts == oparts
    assert launches < len(raws), launches


def test_xz_split_unarchive_decodes_blocks_as_one_batch(gpu, oracle):
    # CHECK_NONE: with a per-block check, every stream costs a check launch on the batched and the sequential path alike
    rng = random.Random(33)
    raws = [H.textlike(rng.randrange(1, 60000), 500 + i) for i in range(24)]
    data = b"".join(lzma.compress(r, format=lzma.FORMAT_XZ, check=lzma.CHECK_NONE) + bytes(4 * (i % 2))
                    for i, r in enumerate(raws))
    ost, oparts, _ = oracle.xz_split_unarchive(data)
    assert ost == 0 and oparts == raws
    parts, launches = _launches(gpu.XZArchive.splitUnarchive, data)
    assert parts == oparts
    assert launches < len(raws), launches
