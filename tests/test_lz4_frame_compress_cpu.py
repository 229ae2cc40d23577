"""swc_lz4_frame_compress_max_bytes against the frames of the CPU restatement of LZ4.compress: never below a frame, equal to
the frame when every block is stored."""
import random

import pytest

import lz4c_cases as K


@pytest.fixture(scope="module")
def oc():
    import swco_lz4c
    swco_lz4c.lib()
    return swco_lz4c


def _bound(n, bs, bc, cc, cs, dict_id):
    from swcompression_b200 import LZ4
    return LZ4.max_compressed_size(n, blockChecksums=bc, contentChecksum=cc, contentSize=cs, blockSize=bs, dictionaryID=dict_id)


FLAGS = [(ind, bc, cc, cs) for ind in (True, False) for bc in (False, True) for cc in (False, True) for cs in (False, True)]


@pytest.mark.parametrize("bs", K.SWEEP_BLOCK_SIZES)
def test_bound_covers_option_sweep(oc, bs):
    inputs = K.frame_inputs() + [("strings", s) for s in K.STRINGS] + [("tricky", K.TRICKY)]
    for name, data in inputs:
        for ind, bc, cc, cs in FLAGS:
            for dict_id in (None, 9):
                if bs == 1024 and len(data) > 80000 and (bc, cc, cs, dict_id) != (True, True, True, None):
                    continue
                st, frame, _ = oc.lz4_compress(data, independentBlocks=ind, blockChecksums=bc, contentChecksum=cc,
                                               contentSize=cs, blockSize=bs, dictionaryID=dict_id)
                assert st == 0
                assert len(frame) <= _bound(len(data), bs, bc, cc, cs, dict_id), (name, bs, ind, bc, cc, cs, dict_id)


@pytest.mark.parametrize("bs", K.SWEEP_BLOCK_SIZES)
def test_bound_is_reached_when_every_block_is_stored(oc, bs):
    rng = random.Random(5)
    for n in (0, 1, 100, bs - 1, bs, bs + 1, 70001):
        if n > 300000:
            continue
        data = bytes(rng.getrandbits(8) for _ in range(n))
        for ind, bc, cc, cs in FLAGS:
            st, frame, _ = oc.lz4_compress(data, independentBlocks=ind, blockChecksums=bc, contentChecksum=cc, contentSize=cs,
                                           blockSize=bs, dictionaryID=3)
            assert st == 0 and len(frame) == _bound(n, bs, bc, cc, cs, 3), (n, bs, ind, bc, cc, cs)


def test_bound_formula_and_invalid_block_size():
    from swcompression_b200 import LZ4
    assert LZ4.max_compressed_size(0) == 7 + 4 + 4
    assert LZ4.max_compressed_size(10, blockSize=4, blockChecksums=True, contentSize=True, dictionaryID=1) == \
        7 + 8 + 4 + 10 + 3 * 8 + 4 + 4
    for bs in (0, -5, (4 << 20) + 1):
        assert LZ4.max_compressed_size(100, blockSize=bs) == 0
