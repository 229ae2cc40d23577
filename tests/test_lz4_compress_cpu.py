"""The CPU restatement of LZ4.compress (oracle/lz4_compress.c, LZ4+Compress.swift:16-298) against frames derived by hand
from the Swift source, against a plain-Python statement of the block parse, and through two decoders."""
import ctypes as C
import random
import struct

import pytest

import helpers as H
import lz4c_cases as K
from oracle_xxh import xxh32

MAGIC = b"\x04\x22\x4D\x18"


@pytest.fixture(scope="module")
def oc():
    """the CPU restatement of LZ4+Compress.swift (oracle/swco_lz4c.py)"""
    import swco_lz4c
    swco_lz4c.lib()
    return swco_lz4c


def frame(blocks, data, independent=True, block_ck=False, content_ck=True, content_size=False, bd=0x70):
    """LZ4+Compress.swift:54-151 written out: `blocks` are (payload, stored) pairs"""
    desc = bytes([0x40 | (0x20 if independent else 0) | (0x10 if block_ck else 0) | (0x08 if content_size else 0) |
                  (0x04 if content_ck else 0), bd])
    if content_size:
        desc += struct.pack("<Q", len(data))
    out = MAGIC + desc + bytes([(xxh32(desc) >> 8) & 0xFF])
    for payload, stored in blocks:
        out += struct.pack("<I", len(payload) | (0x80000000 if stored else 0)) + payload
        if block_ck:
            out += struct.pack("<I", xxh32(payload))
    out += b"\0\0\0\0"
    if content_ck:
        out += struct.pack("<I", xxh32(data))
    return out


# raw blocks derived by hand from compress(block:_:): no match can start in the last 11 bytes, so inputs shorter than
# 12 bytes and inputs without a repeated 4-byte key are one literal-only sequence
HAND_BLOCKS = {
    b"ban": b"\x30ban",
    b"banana": b"\x60banana",
    b"abaaba": b"\x60abaaba",
    b"abracadabra": b"\xb0abracadabra",
    b"cabbage": b"\x70cabbage",
    b"baabaabac": b"\x90baabaabac",
    # i=1 finds "AAAA" at 0 (distance 1) and extends to 6 bytes; the 8 bytes left are literals
    b"AAAAAAABBBBCCCD": b"\x12A\x01\x00\x80BBBBCCCD",
    b"AAAAAAA": b"\x70AAAAAAA",
    b"qwertyuiopasdfghjklzxcvbnmQWERTYUIOPASDFGHJKLZXCVBNM1234567890":
        b"\xf0\x2f" + b"qwertyuiopasdfghjklzxcvbnmQWERTYUIOPASDFGHJKLZXCVBNM1234567890",
    bytes(range(256)): b"\xf0\xf1" + bytes(range(256)),
}
# i=5 finds " -C " at 2 (distance 3) and extends to 5 bytes; i=10 and 11 find nothing; the last 11 bytes are literals
TRICKY_BLOCK = b"\x51" + K.TRICKY[:5] + b"\x03\x00" + b"\xb0" + K.TRICKY[10:]


@pytest.mark.parametrize("data", K.STRINGS, ids=lambda d: d[:12].hex())
def test_reference_strings(oc, data):                         # LZ4CompressionTests.swift:21-48
    assert oc.lz4_block_compress(data) == (0, HAND_BLOCKS[data], None)
    blk = HAND_BLOCKS[data]
    stored = len(blk) > len(data)                                 # :112: a literal-only block is always longer
    assert oc.lz4_compress(data) == (0, frame([(data if stored else blk, stored)], data), None)
    assert stored == (data != b"AAAAAAABBBBCCCD")
    assert K.py_block(data) == HAND_BLOCKS[data]


def test_tricky_sequence(oracle, oc):                                 # LZ4CompressionTests.swift:162-171
    expected = frame([(TRICKY_BLOCK, False)], K.TRICKY, independent=False, block_ck=True, content_size=True)
    assert oc.lz4_compress(K.TRICKY, **K.TRICKY_OPTS) == (0, expected, None)
    assert oracle.lz4_decompress(expected)[:2] == (0, K.TRICKY)


def test_empty_input(oc):
    # no blocks at all (the stride over an empty range), then EndMark and the checksum of nothing
    assert oc.lz4_compress(b"") == (0, frame([], b""), None)
    assert oc.lz4_compress(b"", dictionary=b"ab")[0] == 0       # a short dictionary only traps once a block uses it
    # the raw block of nothing is the single token 0x00 (the assert at :261 is compiled out of release builds)
    assert oc.lz4_block_compress(b"") == (0, b"\x00", None)


def test_stored_blocks_and_block_sizes(oc):
    rng = random.Random(3)
    data = bytes(rng.getrandbits(8) for _ in range(3000))
    # random bytes: every block is longer compressed, so each is stored raw (:112-125); 1 024-byte blocks, BD 0x40
    blocks = [(data[i:i + 1024], True) for i in range(0, 3000, 1024)]
    expected = frame(blocks, data, block_ck=True, content_size=True, bd=0x40)
    assert oc.lz4_compress(data, True, True, True, True, 1024) == (0, expected, None)
    for bs, bd in ((64 << 10, 0x40), ((64 << 10) + 1, 0x50), (256 << 10, 0x50), ((256 << 10) + 1, 0x60), (1 << 20, 0x60),
                   ((1 << 20) + 1, 0x70), (4 << 20, 0x70)):
        assert oc.lz4_compress(b"x", blockSize=bs)[1][5] == bd                      # :66-76


def test_equal_size_stays_compressed(oc):
    data = K.compressible_equal_size()
    blk = oc.lz4_block_compress(data)[1]
    assert len(blk) == len(data) and blk != data
    assert oc.lz4_compress(data)[1] == frame([(blk, False)], data)


def test_dictionary_id(oc):
    expected_desc = bytes([0x65, 0x70]) + struct.pack("<I", 20000)
    out = oc.lz4_compress(b"hello", dictionary=b"", dictionaryID=20000)[1]
    assert out[4:10] == expected_desc and out[10] == (xxh32(expected_desc) >> 8) & 0xFF


@pytest.mark.parametrize("kwargs", [dict(blockSize=0), dict(blockSize=-1), dict(blockSize=(4 << 20) + 1),
                                    dict(dictionary=b"a"), dict(dictionary=b"ab"), dict(dictionary=b"abc"),
                                    dict(independentBlocks=False, blockSize=3), dict(independentBlocks=False, blockSize=1)])
def test_reference_traps(oc, kwargs):
    assert oc.lz4_compress(b"abcdefgh", **kwargs)[0] == 2                         # SWC_ERR_REFERENCE_TRAP


def test_single_short_dependent_block_does_not_trap(oc):
    # a dependent frame with 3-byte blocks traps only when a second block takes the first one as its dictionary
    assert oc.lz4_compress(b"abc", independentBlocks=False, blockSize=3)[0] == 0


@pytest.mark.parametrize("name,block,dictionary,variant", K.edge_blocks(), ids=lambda v: v if isinstance(v, str) else None)
def test_edge_blocks(oracle, oc, name, block, dictionary, variant):
    ref = K.py_block(block, dictionary)
    assert oc.lz4_block_compress(block, dictionary) == (0, ref, None)
    if variant is not None:                                       # the case tells the reference from its near-miss
        assert K.py_block(block, dictionary, variant) != ref
    assert oracle.lz4_block(ref, dictionary)[:2] == (0, block)


def _lz4_safe(block, size, dictionary=b""):
    L = H.liblz4()
    dst = C.create_string_buffer(max(size, 1))
    if dictionary:
        n = L.LZ4_decompress_safe_usingDict(block, dst, len(block), size, dictionary, len(dictionary))
    else:
        n = L.LZ4_decompress_safe(block, dst, len(block), size)
    return dst.raw[:n] if n >= 0 else None


def test_random_options_round_trip(oracle, oc):                       # LZ4CompressionTests.swift:85-110
    rng = random.Random(20240601)
    for name, data in K.frame_inputs():
        for _ in range(6):
            opts = dict(independentBlocks=rng.random() < .5, blockChecksums=rng.random() < .5,
                        contentChecksum=rng.random() < .5, contentSize=rng.random() < .5,
                        blockSize=rng.choice(K.SWEEP_BLOCK_SIZES))
            st, out, _ = oc.lz4_compress(data, **opts)
            assert st == 0
            assert oracle.lz4_decompress(out)[:2] == (0, data), (name, opts)


def test_blocks_decode_with_liblz4(oc):
    for name, data in K.frame_inputs():
        for off in range(0, len(data), 65536):
            blk = data[off:off + 65536]
            enc = oc.lz4_block_compress(blk)[1]
            assert _lz4_safe(enc, len(blk)) == blk, name
            prev = data[max(0, off - 65536):off]
            if len(prev) >= 4:
                enc = oc.lz4_block_compress(blk, prev)[1]
                assert _lz4_safe(enc, len(blk), prev) == blk, name
    for name, block, dictionary, _ in K.edge_blocks():
        assert _lz4_safe(oc.lz4_block_compress(block, dictionary)[1], len(block), dictionary) == block, name


def test_small_dict_fixture(oracle, oc):                               # LZ4CompressionTests.swift:141-160
    d = H.fixture("LZ4/lz4_small_dict")
    meta = K.COMPRESS_MANIFEST["dictionaries"]["LZ4/lz4_small_dict"]
    import hashlib
    assert len(d) == meta["size"] == 1024 and hashlib.sha256(d).hexdigest() == meta["sha256"]
    data = dict(K.frame_inputs())["text"]
    for independent in (True, False):
        st, out, _ = oc.lz4_compress(data, independent, True, True, True, 256 * 1024, d)
        assert st == 0 and oracle.lz4_decompress(out, d)[:2] == (0, data)
