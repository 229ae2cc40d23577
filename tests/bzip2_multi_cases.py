"""A named catalogue of whole multi-stream .bz2 files for the block-parallel multi-stream batch
(swc_bzip2_multi_decompress_batch, Batch codec 'bzip2_multi'): 0 bytes, one stream and 2 to 300 streams, levels 1 and 9
mixed, empty 14-byte streams between and after real ones (and a file of empty streams only), multi-block streams next to
single-block ones, an end magic that ends on a byte (no padding), non-zero padding bits, trailing bytes (zeros, "BZ",
"BZh0", "BZx9"), a wrong block CRC or combined CRC in stream k, a decode error in a later stream, and block / end magic
look-alikes spelled into payloads, among them whole valid blocks that decode to bytes of their own.  Streams come from tests/bzip2_writer.py and from Python's bz2.compress.

case.status is what BZip2.multiDecompress returns, read off the Swift source (BZip2.swift:40-95) and the way each case is
built.  expect() gives the reference's full answer from the oracle."""
import bz2
import functools
import random

import bzip2_cases as D
import helpers as H
from bzip2_writer import Block, BZip2Writer, bwt_of

OK, WRONG_MAGIC, WRONG_VERSION, WRONG_LEVEL, RANDOMISED, WRONG_CRC = D.OK, D.WRONG_MAGIC, D.WRONG_VERSION, D.WRONG_LEVEL, D.RANDOMISED, D.WRONG_CRC
EMPTY = bz2.compress(b"")                      # 14 bytes: header, end magic, combined CRC 0, padding
BLOCK_MAGIC, END_MAGIC = format(0x314159265359, "048b"), format(0x177245385090, "048b")


class Case:
    """libbz2: Python's bz2 decodes the file as the reference does (the spelled look-alike blocks use code tables libbzip2
    does not take)"""
    __slots__ = ("name", "data", "status", "libbz2")

    def __init__(self, name, data, status=OK, libbz2=True):
        self.name, self.data, self.status, self.libbz2 = name, bytes(data), status, libbz2


def text(n, seed):
    return H.textlike(n, seed)


def written(texts, level=9, crc=None, combined=None, randomised_at=None):
    """a writer stream of one block per text; `crc` = {block index: wrong CRC}; `combined`: a wrong combined CRC;
    `randomised_at`: a block index whose randomised bit is set (a decode error)"""
    w = BZip2Writer(level)
    for k, t in enumerate(texts):
        bad = randomised_at == k
        w.block(Block(*bwt_of(t), crc=(crc or {}).get(k), randomised=1 if bad else 0), model=not bad)
    return w.finish(combined)[0]


def aligned_stream(seed=0):
    """a writer stream whose end CRC ends on a byte boundary (no padding bits)"""
    rng = random.Random(seed)
    for n in range(40, 400):
        w = BZip2Writer(9)
        w.block(Block(*bwt_of(bytes(rng.choice(b"abcdefgh") for _ in range(n)))))
        data, nbits = w.finish()
        if nbits % 8 == 0:
            return data
    raise AssertionError("no byte-aligned stream found")


def padded_with_ones(texts):
    """a writer stream with its padding bits (behind the combined CRC) set to 1"""
    w = BZip2Writer(9)
    for t in texts:
        w.block(Block(*bwt_of(t)))
    data, nbits = w.finish()
    assert nbits % 8, "the stream has no padding bits"
    return data[:-1] + bytes([data[-1] | ((1 << (-nbits % 8)) - 1)])


def lookalike_stream(pattern, k, seed):
    """a writer stream of three blocks, the middle one carrying `pattern` k (mod 8) bits into the stream"""
    rng = random.Random(seed)
    w = BZip2Writer(9)
    w.block(Block(*bwt_of(bytes(rng.choice(b"abcd") for _ in range(300)))))
    D.spelled_block(w, pattern, k)
    w.block(Block(*bwt_of(bytes(rng.choice(b"abcd") for _ in range(200)))))
    return w.finish()[0]


def valid_cases():
    t = [text(3000 + 700 * i, 900 + i) for i in range(8)]
    s9 = [bz2.compress(x, 9) for x in t]
    s1 = [bz2.compress(x, 1) for x in t]
    multi_block = bz2.compress(text(260_000, 77), 1)           # three 100 kB blocks
    out = [
        Case("zero_bytes", b""),
        Case("one_stream", s9[0]),
        Case("two_streams", s9[0] + s9[1]),
        Case("eight_streams", b"".join(s9)),
        Case("levels_1_and_9_mixed", b"".join(a if i % 2 else b for i, (a, b) in enumerate(zip(s1, s9)))),
        Case("empty_between_and_after", s9[0] + EMPTY + s9[1] + EMPTY + EMPTY),
        Case("empty_first", EMPTY + s9[2]),
        Case("empty_only", EMPTY * 5),
        Case("one_empty", EMPTY),
        Case("multi_block_next_to_single", s9[3] + multi_block + s1[4]),
        Case("writer_streams", written([text(500, 1), text(800, 2)]) + written([text(300, 3)], level=1)
             + written([text(200, 4), text(100, 5), text(50, 6)])),
        Case("end_on_a_byte", aligned_stream(1) + aligned_stream(2) + s9[5]),
        Case("padding_bits_set", padded_with_ones([text(700, 8)]) + padded_with_ones([text(333, 9), text(90, 10)]) + s1[7]),
        Case("three_hundred_streams", b"".join(bz2.compress(text(50 + i % 97, 3000 + i), 1 + i % 9) for i in range(300))),
    ]
    for k in range(0, 8, 3):
        out.append(Case(f"block_lookalike_bit_{k}", s9[0] + lookalike_stream(BLOCK_MAGIC, k, k) + s9[1], libbz2=False))
        out.append(Case(f"end_lookalike_bit_{k}", lookalike_stream(END_MAGIC, k, 10 + k) + EMPTY + s9[2], libbz2=False))
    return out


def tail_cases():
    s = bz2.compress(text(2000, 5), 9) + bz2.compress(text(1500, 6), 9)
    return [
        Case("trailing_1_zero", s + b"\0", WRONG_MAGIC),
        Case("trailing_2_zeros", s + b"\0\0", WRONG_MAGIC),
        Case("trailing_3_zeros", s + b"\0\0\0", WRONG_MAGIC),
        Case("trailing_5_zeros", s + b"\0" * 5, WRONG_MAGIC),
        Case("trailing_BZ", s + b"BZ", WRONG_MAGIC),
        Case("trailing_BZh0", s + b"BZh0", WRONG_LEVEL),
        Case("trailing_BZx9", s + b"BZx9", WRONG_VERSION),
        Case("trailing_header_only", s + b"BZh9", WRONG_MAGIC),
    ]


def damage_cases():
    good = [written([text(600 + 100 * i, 40 + i), text(300, 50 + i)]) for i in range(4)]
    out = []
    for k in (0, 2, 3):
        bad_block = written([text(600 + 100 * k, 40 + k), text(300, 50 + k)], crc={1: 0x12345678})
        bad_total = written([text(600 + 100 * k, 40 + k), text(300, 50 + k)], combined=0xDEADBEEF)
        out.append(Case(f"block_crc_in_stream_{k}", b"".join(good[:k] + [bad_block] + good[k + 1:]), WRONG_CRC))
        out.append(Case(f"combined_crc_in_stream_{k}", b"".join(good[:k] + [bad_total] + good[k + 1:]), WRONG_CRC))
    bad = written([text(400, 60), text(300, 61)], randomised_at=1)
    out.append(Case("decode_error_in_stream_2", good[0] + good[1] + bad + good[2], RANDOMISED))
    out.append(Case("cut_last_stream", good[0] + good[1] + good[2][:-5], WRONG_MAGIC))
    return out


@functools.lru_cache(maxsize=None)
def cases():
    return tuple(valid_cases() + tail_cases() + damage_cases())


def three_stream_file():
    """a three-stream file under 4 KiB: a writer stream, an empty stream and a bz2.compress stream"""
    return written([text(400, 90), text(200, 91)]) + EMPTY + bz2.compress(text(900, 92), 9)


def cuts():
    """every byte cut of the three-stream file: (name, data) with data a proper prefix"""
    f = three_stream_file()
    assert len(f) < 4096
    return [(f"three_streams cut {k}", f[:k]) for k in range(len(f))]


def expect(oracle, data):
    """the reference's answer: (status, output, stream ends, stream starts); output and table are empty unless the status
    is OK or wrongCRC (then the failing stream is the table's last entry)"""
    st, parts, whole = oracle.bzip2_multi_decompress(data)
    if st not in (OK, WRONG_CRC):
        return st, b"", [], []
    ends, starts, off, total = [], [], 0, 0
    for p in parts:
        starts.append(off)
        s1, out, used = oracle.bzip2_decompress(data[off:])
        assert s1 == OK and out == p
        off += (used + 7) // 8
        total += len(p)
        ends.append(total)
    if st == WRONG_CRC:
        starts.append(off)
        ends.append(len(whole))
    return st, whole, ends, starts
