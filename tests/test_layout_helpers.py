"""CPU checks of the hostile-layout helpers behind tests/test_gpu_layout.py: a fixture that did not put foreign bytes next
to its units, or whose cut units decode the same with and without their rest, would prove nothing on the GPU."""
import random

import numpy as np
import pytest

import helpers as H


def _coverage(buf, offs, units):
    """mask of the bytes that belong to a unit, its head or its tail"""
    mask = np.zeros(len(buf), dtype=bool)
    for o, u in zip(offs.tolist(), units):
        head, tail = len(u.head or b""), len(u.tail or b"")
        mask[o - head:o + len(u.data) + tail] = True
    return mask


@pytest.mark.parametrize("name", sorted(H.LAYOUT_SETS))
def test_pack_hostile_places_units_between_foreign_bytes(name):
    _, make = H.LAYOUT_SETS[name]
    units = make()
    buf, offs, lens = H.pack_hostile([u.data for u in units], random.Random(1), [u.head for u in units], [u.tail for u in units])
    assert set((offs % 16).tolist()) == set(range(16))
    gaps = [int(offs[i]) - len(units[i].head or b"") - (int(offs[i - 1]) + int(lens[i - 1]) + len(units[i - 1].tail or b""))
            for i in range(1, len(units))]
    assert min(gaps) == 0 and max(gaps) >= 16                       # tight neighbours and filler both occur
    for o, u in zip(offs.tolist(), units):
        assert bytes(buf[o:o + len(u.data)]) == u.data
        if u.head:
            assert bytes(buf[o - len(u.head):o]) == u.head
        if u.tail:
            assert bytes(buf[o + len(u.data):o + len(u.data) + len(u.tail)]) == u.tail
    filler = buf[~_coverage(buf, offs, units)]
    assert filler.size and (filler != 0).all()
    assert (buf[-H.GUARD:] == 0xFF).all()
    assert sum(u.tail is not None for u in units) >= 10 and any(u.head is not None for u in units) == (name != "deflate_shifted")


@pytest.mark.parametrize("name", sorted(H.LAYOUT_SETS))
def test_cut_units_decode_differently_without_their_neighbours(oracle, name):
    """Each cut unit's answer from its own bytes differs from the answer with its head / tail in place, and every whole
    valid unit decodes to the bytes it was made from."""
    codec, make = H.LAYOUT_SETS[name]
    valid = 0
    for u in make():
        own = H.layout_oracle(codec, oracle, u.data, u.aux)
        if u.head is not None or u.tail is not None:
            whole = H.layout_oracle(codec, oracle, (u.head or b"") + u.data + (u.tail or b""), u.aux)
            assert whole[0] == 0 and own[:2] != whole[:2], (name, len(u.data), own[0])
        if u.raw is not None:
            assert own[0] == 0 and own[1] == u.raw
            valid += 1
    assert valid >= 20


@pytest.mark.parametrize("shifts", [False, True])
def test_malformed_code_sets_include_accepted_units(oracle, shifts):
    units = H.layout_malformed_deflate(random.Random(102 + 2 * shifts), 60, shifts)
    accepted = sum(H.layout_oracle("deflate", oracle, u.data, u.aux)[0] == 0 for u in units)
    assert 0 < accepted < len(units)


def test_lz4_sequences_cross_the_warp_copy_threshold(oracle):
    units = H.lz4_dictionary_units(random.Random(3), 24, H.LZ4_DICTIONARY)
    for u in units[:-2]:
        if u.raw is not None:
            assert oracle.lz4_block(u.data, H.LZ4_DICTIONARY)[1] == u.raw
    st_first, st_before = (oracle.lz4_block(u.data, H.LZ4_DICTIONARY)[0] for u in units[-2:])
    assert st_first == 0 and st_before != 0
    blk, raw = H.lz4_block_from_sequences([(b"abcdefgh" * 8, 65, 1), (b"x" * 63, 64, 16), (b"y" * 65, 63, 300)], b"z" * 12)
    assert oracle.lz4_block(blk) == (0, raw, None)


def test_fenced_layout_caps_and_guards():
    sizes = [1000 + 37 * i for i in range(96)] + [None] * 4
    offs, caps, total = H.fenced_layout(sizes)
    assert (offs % 16 == 0).all() and offs[0] == H.GUARD
    assert set((caps % 16).tolist()) == set(range(16))
    known = np.array(sizes[:96])
    delta = caps[:96].astype(np.int64) - known
    assert (delta == 0).any() and set((-delta[delta < 0]).tolist()) == set(range(1, 16)) and set(delta[delta > 0].tolist()) == set(range(1, 16))
    ends = offs + caps
    assert (offs[1:] > ends[:-1]).all() and total - int(ends[-1]) >= H.GUARD


def test_fence_violations_finds_a_stray_byte():
    offs, caps, total = H.fenced_layout([100, 200, 300])
    out = np.full(total, H.SENTINEL, dtype=np.uint8)
    out[int(offs[1]):int(offs[1]) + int(caps[1])] = 7             # inside a region: allowed
    assert H.fence_violations(out, offs, caps).size == 0
    out[int(offs[1]) + int(caps[1])] = 7                          # first byte behind it
    out[0] = 0
    assert H.fence_violations(out, offs, caps).tolist() == [0, int(offs[1]) + int(caps[1])]
