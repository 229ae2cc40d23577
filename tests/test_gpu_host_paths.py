"""The host-side retry paths of the single-unit decoders and of the LZ4 frame layer: outputs far larger than the first
capacity guess must come out equal to the oracle's, through every API that reaches each path."""
import bz2
import lzma
import struct
import zlib

import pytest

import helpers as H

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def gpu():
    import torch
    assert torch.cuda.is_available()
    import swcompression_b200 as S
    return S


def outcome(gpu, fn, data):
    try:
        return 0, fn(data)
    except gpu.SWCompressionError as e:
        return e.code, e.payload


# ---- Deflate: the first capacity is 4 x input + 64 KiB; the retry takes the exact size the counting pass reports ----
RUN = bytes([0x61]) * (8 << 20)


def test_deflate_exact_size_retry(gpu, oracle):
    raw = zlib.compressobj(9, zlib.DEFLATED, -15)
    raw = raw.compress(RUN) + raw.flush()
    assert len(RUN) > 4 * len(raw) + 65536
    ost, oout, oused = oracle.deflate_decompress(raw)
    assert ost == 0 and oout == RUN
    assert gpu.Deflate.decompress_from(raw, 0) == (RUN, oused)
    gz = zlib.compressobj(9, zlib.DEFLATED, 31)
    gz = gz.compress(RUN) + gz.flush()
    assert oracle.gzip_unarchive(gz)[:2] == (0, RUN)
    assert gpu.GzipArchive.unarchive(gz) == RUN
    zl = zlib.compress(RUN, 9)
    assert oracle.zlib_unarchive(zl)[:2] == (0, RUN)
    assert gpu.ZlibArchive.unarchive(zl) == RUN


# ---- BZip2: the first capacity is 16 x input + 1 MiB, then x4 per attempt ----
def test_bzip2_growth(gpu, oracle):
    raw = bytes(8 << 20)                                      # one block: RLE1 packs the zeros far below 900 000 bytes
    data = bz2.compress(raw, 9)
    assert len(raw) > 4 * (16 * len(data) + (1 << 20))        # a third attempt
    ost, oout, _ = oracle.bzip2_decompress(data)
    assert ost == 0 and oout == raw
    assert gpu.BZip2.decompress(data) == raw


# ---- LZMA: the first capacity is 8 x input + 1 MiB, then x4 per attempt ----
BIG = bytes(6 << 20)


def third_attempt(data):
    return len(BIG) > 4 * (8 * len(data) + (1 << 20))


def test_lzma2_growth(gpu, oracle):
    l2 = bytes([18]) + lzma.compress(BIG, format=lzma.FORMAT_RAW, filters=[{"id": lzma.FILTER_LZMA2, "preset": 6, "dict_size": 1 << 20}])
    assert third_attempt(l2)
    ost, oout, oused = oracle.lzma2_decompress(l2)
    assert ost == 0 and oout == BIG
    assert gpu.LZMA2.decompress(l2) == BIG


def test_lzma_raw_unknown_size_growth(gpu, oracle):
    raw = lzma.compress(BIG, format=lzma.FORMAT_RAW, filters=[{"id": lzma.FILTER_LZMA1, "lc": 3, "lp": 0, "pb": 2, "dict_size": 1 << 20}])
    assert third_attempt(raw)
    ost, oout, _ = oracle.lzma_decompress_raw(raw, 3, 0, 2, 1 << 20)
    assert ost == 0 and oout == BIG
    props = gpu.LZMAProperties(lc=3, lp=0, pb=2, dictionarySize=1 << 20)
    assert gpu.LZMA.decompress(raw, props) == BIG


def test_xz_single_block_without_sizes_growth(gpu, oracle):
    xz = lzma.compress(BIG, check=lzma.CHECK_CRC64)
    assert xz[13] & 0xC0 == 0                                 # block flags: neither size field is present
    assert third_attempt(xz)
    assert oracle.xz_unarchive(xz)[:2] == (0, BIG)
    assert gpu.XZArchive.unarchive(xz) == BIG
    assert gpu.XZArchive.splitUnarchive(xz) == [BIG]


# ---- LZ4 frames: a block may decode past the frame's maximum block size; the first attempt sizes for that maximum ----
def lz4_frame(blocks_raw, independent, content_checksum):
    import oracle_xxh
    desc = bytes([0x40 | (0x20 if independent else 0) | (0x04 if content_checksum else 0), 0x40])      # 64 KiB blocks
    out = bytearray(struct.pack("<I", 0x184D2204) + desc + bytes([(oracle_xxh.xxh32(desc) >> 8) & 0xFF]))
    for raw in blocks_raw:
        comp = H.lz4_block_compress(raw)
        assert len(comp) <= 65536
        out += struct.pack("<I", len(comp)) + comp
    out += struct.pack("<I", 0)
    if content_checksum:
        out += struct.pack("<I", oracle_xxh.xxh32(b"".join(blocks_raw)))
    return bytes(out)


@pytest.mark.parametrize("independent", [True, False])
@pytest.mark.parametrize("content_checksum", [True, False])
def test_lz4_block_past_max_block_size(gpu, oracle, independent, content_checksum):
    blocks = [H.textlike(30000, 71), bytes(300000), H.textlike(65536, 72), b"\x07" * 200000, H.textlike(100, 73)]
    frame = lz4_frame(blocks, independent, content_checksum)
    ost, oout, _ = oracle.lz4_decompress(frame)
    assert (ost, oout) == (0, b"".join(blocks))
    assert outcome(gpu, gpu.LZ4.decompress, frame) == (ost, oout)
    two = frame + lz4_frame(blocks[:2], independent, content_checksum)
    mst, mparts, _ = oracle.lz4_multi_decompress(two)
    assert outcome(gpu, gpu.LZ4.multiDecompress, two) == (mst, mparts)
