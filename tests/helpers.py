"""Shared test helpers: golden fixtures, synthetic corpora, a Python LsbBitWriter (BitByteData semantics)."""
import ctypes as C
import json
import os
import random
import struct
import zlib

import numpy as np

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")

with open(os.path.join(GOLDEN, "manifest.json")) as _f:
    MANIFEST = json.load(_f)


def answer(name):
    a = MANIFEST["answers"][name]
    if "literal" in a:
        return a["literal"].encode().decode("unicode_escape").encode("latin1")
    return bytes(a["zeros"])


def fixture(rel):
    with open(os.path.join(GOLDEN, rel), "rb") as f:
        return f.read()


def fixtures(prefix):
    return [(rel, meta["answer"]) for rel, meta in sorted(MANIFEST["fixtures"].items()) if rel.startswith(prefix)]


class LsbBitWriter:
    """BitByteData.LsbBitWriter: bits fill each byte from bit 0 upward; numbers are written LSB first."""

    def __init__(self):
        self.bits = []

    def write_bits(self, bits):
        self.bits.extend(bits)

    def write_number(self, value, count):
        for i in range(count):
            self.bits.append((value >> i) & 1)

    def align(self):
        while len(self.bits) % 8:
            self.bits.append(0)

    @property
    def data(self):
        self.align()
        out = bytearray()
        for i in range(0, len(self.bits), 8):
            out.append(sum(b << k for k, b in enumerate(self.bits[i:i + 8])))
        return bytes(out)


# literal round-trip vectors of the reference's compression tests (DeflateCompressionTests.swift:7-83,
# BZip2CompressionTests.swift:11-95, LZ4CompressionTests.swift:11-171)
ROUNDTRIP_STRINGS = [
    b"ban", b"banana", b"abaaba", b"abracadabra", b"cabbage", b"baabaabac", b"AAAAAAABBBBCCCD", b"AAAAAAA",
    b"abcdefghijklmnopqrstuvwxyzABCDEFGHIJKLMNOPQRSTUVWXYZ0123456789", bytes(range(256)), b"", b"a",
    b"Hello, World!\n", b"the quick brown fox jumps over the lazy dog " * 40,
]


def textlike(n, seed):
    """SURVEY.md §8(d) corpus: order-1 Markov over a 64-symbol Zipf(1.2) alphabet + ~30 % back-references."""
    rng = np.random.Generator(np.random.PCG64(seed))
    ranks = np.arange(1, 65, dtype=np.float64)
    p = ranks ** -1.2
    p /= p.sum()
    alphabet = np.frombuffer(b"etaoinshrdlucmfwypvbgkjqxz ETAOINSHRDLUCMFWYPVBGKJQXZ.,;:!?-'\"()\n", dtype=np.uint8)[:64]
    # order-1 flavour: each previous symbol rotates the Zipf ranking
    base = rng.choice(64, size=n, p=p)
    prev = np.concatenate([[0], base[:-1]])
    sym = (base + (prev * 7)) % 64
    out = alphabet[sym].copy()
    # back-references
    i = 64
    while i < n - 70:
        if rng.random() < 0.12:
            ln = int(rng.integers(3, 65))
            dist = int(rng.integers(1, min(i, 32768) + 1))
            for k in range(ln):
                out[i + k] = out[i + k - dist]
            i += ln
        else:
            i += int(rng.integers(1, 12))
    return out.tobytes()


def raw_deflate(data, level=6, mem_level=9):
    c = zlib.compressobj(level, zlib.DEFLATED, -15, mem_level)
    return c.compress(data) + c.flush()


_lz4 = None


def liblz4():
    global _lz4
    if _lz4 is None:
        _lz4 = C.CDLL("liblz4.so.1")
        _lz4.LZ4_compressBound.restype = C.c_int
        _lz4.LZ4_compress_default.restype = C.c_int
        _lz4.LZ4_compress_default.argtypes = [C.c_char_p, C.c_void_p, C.c_int, C.c_int]
    return _lz4


def lz4_block_compress(data):
    L = liblz4()
    cap = L.LZ4_compressBound(len(data))
    dst = C.create_string_buffer(max(cap, 16))
    n = L.LZ4_compress_default(data, dst, len(data), cap)
    assert n > 0 or len(data) == 0
    return dst.raw[:n]


def lz4_block_from_sequences(seqs, last, prefix=b""):
    """Raw LZ4 block built by hand from (literals, match length, offset) sequences and the final literal run.
    -> (block, decoded bytes); `prefix` is the dictionary the offsets may reach into."""
    def ext(v):
        return b"\xFF" * (v // 255) + bytes([v % 255])
    blk, out = bytearray(), bytearray(prefix)
    for lit, mlen, off in seqs:
        blk.append(min(len(lit), 15) << 4 | min(mlen - 4, 15))
        if len(lit) >= 15:
            blk += ext(len(lit) - 15)
        blk += lit
        out += lit
        blk += struct.pack("<H", off)
        if mlen - 4 >= 15:
            blk += ext(mlen - 19)
        for _ in range(mlen):
            out.append(out[-off])
    blk.append(min(len(last), 15) << 4)
    if len(last) >= 15:
        blk += ext(len(last) - 15)
    blk += last
    out += last
    return bytes(blk), bytes(out[len(prefix):])


# ---------------------------------------------------------------------------------------------------------------------
# Hostile batch layouts.  The batched entry points (include/swcgpu.h, "Batch layout") let a unit start at any byte, read
# only in_base[in_off, in_off + in_len) and write only out_base[out_off, out_off + out_cap).  batch.pack_units puts every
# unit on a 16-byte boundary with zeros behind it, which is what a correctly masking kernel sees anyway; these helpers lay
# units out the way ZIP members, gzip members and back-to-back streams really sit, so that a kernel that reads a
# neighbour's bytes or writes past its region gives a different answer.
SENTINEL = 0xA5          # fill of every output buffer before a run
GUARD = 64               # bytes before the first and after the last output region / behind the last input unit


def shifted(data, k, junk):
    """`data` moved up by k bits inside its first byte, the k low bits of that byte being `junk` (the start_bits form)."""
    if k == 0:
        return bytes(data)
    v = (int.from_bytes(data, "little") << k) | (junk & ((1 << k) - 1))
    return v.to_bytes(len(data) + 1, "little")


def pack_hostile(units, rng, heads=None, tails=None, residues=None):
    """Pack `units` into one input buffer with no friendly bytes around them -> (uint8 buffer, offsets u64, lengths u64).

    - heads[i] / tails[i] (bytes or None) sit directly in front of / behind unit i: the rest of the stream a unit was cut
      from, so a kernel reading outside [in_off, in_off + in_len) sees data that changes its answer;
    - the gap in front of a unit (and its head) cycles through three kinds: a run of 0xFF, random non-zero bytes, and none
      at all (the unit follows its neighbour's last byte);
    - units behind a gap start at residues 0, 1, ..., 15 (mod 16) in turn, unless residues[i] asks for one;
    - GUARD bytes of 0xFF follow the last unit, and no byte outside the units, heads and tails is zero."""
    n = len(units)
    heads = heads or [None] * n
    tails = tails or [None] * n
    buf = bytearray(b"\xFF" * 16)
    offs = np.zeros(n, dtype=np.uint64)
    k = 0
    for i, u in enumerate(units):
        head, tail = heads[i] or b"", tails[i] or b""
        kind = i % 3
        want = residues[i] if residues is not None and residues[i] is not None else None
        if kind != 2 or want is not None:
            r = want if want is not None else k % 16
            k += want is None
            gap = (r - len(buf) - len(head)) % 16 or 16
            gap += 16 * rng.randrange(2)
            buf += b"\xFF" * gap if kind == 0 else bytes(rng.randrange(1, 256) for _ in range(gap))
        buf += head
        offs[i] = len(buf)
        buf += u
        buf += tail
    buf += b"\xFF" * GUARD
    lens = np.fromiter((len(u) for u in units), dtype=np.uint64, count=n)
    return np.frombuffer(bytes(buf), dtype=np.uint8).copy(), offs, lens


def fenced_layout(sizes, spare=4096, align=16):
    """Output regions for units that decode to `sizes` bytes (None: unknown, e.g. a damaged unit, which gets `spare` bytes).
    Caps cycle through the exact size, 1..15 bytes short of it (overflow) and 1..15 bytes beyond it; regions start on
    multiples of `align` (a power of two up to 16) and cycle through every such residue mod 16, GUARD bytes in front of
    the first one, at least one byte between two regions and GUARD bytes behind the last one.
    -> (out_off u64, out_cap u64, total buffer bytes)"""
    n = len(sizes)
    offs = np.zeros(n, dtype=np.uint64)
    caps = np.zeros(n, dtype=np.uint64)
    pos = GUARD
    for i, s in enumerate(sizes):
        d = 1 + (i // 3) % 15
        if s is None:
            cap = spare + d
        else:
            cap = s if i % 3 == 0 else max(s - d, 0) if i % 3 == 1 else s + d
        offs[i], caps[i] = pos, cap
        pos = (pos + cap + 1 + 15) // 16 * 16 + (16 if i % 2 else 0) + (i + 1) % (16 // align) * align
    return offs, caps, pos + GUARD


def random_bytes(rng, n):
    return bytes(rng.getrandbits(8) for _ in range(n))


def fence_violations(out, out_off, out_cap, sentinel=SENTINEL):
    """Offsets of bytes outside every [out_off, out_off + out_cap) that are no longer `sentinel`."""
    outside = np.ones(len(out), dtype=bool)
    for o, c in zip(out_off.tolist(), out_cap.tolist()):
        outside[o:o + c] = False
    return np.nonzero(outside & (np.asarray(out) != sentinel))[0]


class LayoutUnit:
    """One unit of a hostile batch: `data` is what the kernel is given, `head` / `tail` the stream bytes around it in memory
    (None: filler), `aux` the per-unit argument (Deflate start bit, LZMA2 dictionary byte, (props, dict size, size) of raw
    LZMA), `raw` the original bytes when `data` is a whole valid stream."""
    __slots__ = ("data", "head", "tail", "aux", "raw")

    def __init__(self, data, head=None, tail=None, aux=0, raw=None):
        self.data, self.head, self.tail, self.aux, self.raw = bytes(data), head, tail, aux, raw


def layout_oracle(codec, oracle, data, aux, dictionary=None):
    """The reference's answer for one unit, from its own bytes only -> (status, output, consumed)."""
    if codec == "deflate":
        return oracle.deflate_decompress(data, aux)
    if codec == "lz4_block":
        return oracle.lz4_block(data, dictionary)
    if codec == "bzip2":
        return oracle.bzip2_decompress(data)
    if codec == "lzma2":
        return oracle.lzma2_decompress_raw(data, aux)
    props, dsz, usz = aux
    return oracle.lzma_decompress_raw(data, props & 255, (props >> 8) & 255, props >> 16, dsz, None if usz < 0 else usz)


def _variants(rng, stream, raw, aux, front=True):
    """the whole stream, the stream cut with its rest behind it, the stream without its first bytes with those in front of
    it, and the stream with one flipped bit"""
    out = [LayoutUnit(stream, aux=aux, raw=raw)]
    if len(stream) > 2:
        c = rng.randrange(1, len(stream) - 1)                # at least two bytes go: the last may hold only zero bits
        out.append(LayoutUnit(stream[:c], tail=stream[c:], aux=aux))
    if front and len(stream) > 16:
        c = rng.randrange(1, min(len(stream) - 1, 24))
        out.append(LayoutUnit(stream[c:], head=stream[:c], aux=aux))
    if stream:
        b = bytearray(stream)
        b[rng.randrange(len(b))] ^= 1 << rng.randrange(8)
        out.append(LayoutUnit(b, aux=aux))
    return out


def layout_deflate(rng, count, max_raw=12000, shifts=False):
    """Ragged Deflate streams (dynamic, fixed, stored and Huffman-only blocks, empty input) and their cut / damaged forms;
    with `shifts`, stream j starts k = j % 8 junk bits into its first byte (the start_bits form)."""
    units = []
    for j in range(count):
        n = rng.choice([0, 1, 7, 100, 1000, rng.randrange(max_raw + 1), max_raw])
        # a stored block's length field sits on a byte boundary of the reader, so shifted streams keep to coded blocks
        # (compressible input, level >= 1)
        raw = random_bytes(rng, n) if j % 5 == 4 and not shifts else textlike(max(n, 70), 20000 + j)[:n]
        strategy = rng.choice([zlib.Z_DEFAULT_STRATEGY, zlib.Z_FIXED, zlib.Z_HUFFMAN_ONLY])
        c = zlib.compressobj(rng.choice([1, 6, 9] if shifts else [0, 1, 6, 9]), zlib.DEFLATED, -15, 8, strategy)
        s = c.compress(raw) + c.flush()
        k = j % 8 if shifts else 0
        units += _variants(rng, shifted(s, k, rng.getrandbits(8)), raw, k, front=not shifts)
    return units


def layout_malformed_deflate(rng, count, shifts=False):
    """Bit flips inside dynamic-block headers: incomplete and over-subscribed code sets, which the reference accepts and the
    batch decoders hand to the generic slow kernel."""
    units = []
    for j in range(count):
        d = bytearray(raw_deflate(textlike(3000 + (j % 6) * 500, 80 + j % 6)))
        for _ in range(rng.randrange(1, 3)):
            d[rng.randrange(70)] ^= 1 << rng.randrange(8)
        k = j % 8 if shifts else 0
        units.append(LayoutUnit(shifted(d, k, rng.getrandbits(8)), aux=k))
    return units


def lz4_hostile_sequences(rng, count, prefix=b""):
    """Hand-built LZ4 blocks whose literal runs and matches straddle the 64-byte warp-copy threshold (63 / 64 / 65), with
    offsets 1..16 and >= 512; with a `prefix` (dictionary), matches also reach into it, short and long."""
    blocks = []
    for j in range(count):
        seqs, op = [], 0
        first = textlike(1100, 30000 + j)
        seqs.append((first, 4 + j % 3, 1 + j % 16))
        op = len(first) + seqs[0][1]
        for _ in range(rng.randrange(4, 20)):
            lit = textlike(200, rng.randrange(1 << 20))[:rng.choice([0, 1, 4, 15, 16, 63, 64, 65, 200])]
            mlen = rng.choice([4, 5, 18, 19, 63, 64, 65, 300])
            if prefix and rng.random() < 0.4:
                off = op + len(lit) + rng.randrange(1, min(len(prefix), 65535 - op - len(lit)) + 1)
            else:
                off = rng.choice(list(range(1, 17)) + [512, 513, 1000])
            seqs.append((lit, mlen, off))
            op += len(lit) + mlen
        last = textlike(100, 31000 + j)[:rng.choice([12, 15, 63, 64, 65])]
        blocks.append(lz4_block_from_sequences(seqs, last, prefix))
    return blocks


def layout_lz4(rng, count):
    units = []
    for j in range(count):
        n = rng.choice([1, 5, 12, 13, 64, 300, 4000, 20000])
        raw = textlike(max(n, 70), 32000 + j)[:n] if j % 4 else (bytes(n) if j % 8 else random_bytes(rng, n))
        units += _variants(rng, lz4_block_compress(raw), raw, 0)
    for blk, raw in lz4_hostile_sequences(rng, count // 2):
        units += _variants(rng, blk, raw, 0)
    return units


def layout_bzip2(rng, count):
    import bz2
    units = []
    for j in range(count):
        n = rng.choice([0, 1, 5, 256, 1000, 20000, 60000])
        raw = textlike(max(n, 70), 33000 + j)[:n] if j % 3 else (bytes(n) if j % 2 else random_bytes(rng, n))
        units += _variants(rng, bz2.compress(raw, rng.choice([1, 9])), raw, 0)
    return units


def layout_lzma2(rng, count):
    import lzma
    units = []
    for j in range(count):
        n = rng.choice([0, 1, 100, 5000, 30000, 70000])
        raw = textlike(max(n, 70), 34000 + j)[:n] if j % 4 else random_bytes(rng, n)
        s = lzma.compress(raw, format=lzma.FORMAT_RAW, filters=[{"id": lzma.FILTER_LZMA2, "preset": rng.choice([1, 6]), "dict_size": 1 << 20}])
        units += _variants(rng, s, raw, 18)
    return units


def layout_lzma(rng, count):
    """raw LZMA streams with per-unit properties, dictionary size and known / unknown (end marker) size"""
    import lzma
    units = []
    for j in range(count):
        lc, lp, pb = rng.choice([(3, 0, 2), (0, 2, 1), (2, 2, 0), (4, 0, 4), (1, 3, 3), (0, 0, 0)])
        d = rng.choice([1 << 12, 1 << 16, 1 << 20])
        n = rng.choice([0, 1, 100, 5000, 30000])
        raw = textlike(max(n, 70), 35000 + j)[:n]
        alone = lzma.compress(raw, format=lzma.FORMAT_ALONE, filters=[{"id": lzma.FILTER_LZMA1, "lc": lc, "lp": lp, "pb": pb, "dict_size": d}])
        aux = (lc | lp << 8 | pb << 16, d, len(raw) if j % 2 == 0 else -1)
        units += _variants(rng, alone[13:], raw, aux)
    return units


def lz4_dictionary_units(rng, count, dictionary):
    """blocks whose matches reach into `dictionary`, their cut / damaged forms, and one match reaching one byte before it"""
    units = []
    for blk, raw in lz4_hostile_sequences(rng, count, prefix=dictionary):
        units += _variants(rng, blk, raw, 0)
    first = textlike(40, 36000)
    blk, _ = lz4_block_from_sequences([(first, 20, len(first) + len(dictionary))], first[:12], dictionary)
    units.append(LayoutUnit(blk))                          # the match starts at the dictionary's first byte
    bad = bytearray(blk)
    bad[2 + len(first)] += 1                               # token, one length byte, literals: offset + 1 reaches before it
    units.append(LayoutUnit(bad))
    return units


# the fixture sets of tests/test_gpu_layout.py, checked on the CPU by tests/test_layout_helpers.py
LAYOUT_SETS = {
    "deflate": ("deflate", lambda: layout_deflate(random.Random(101), 60) + layout_malformed_deflate(random.Random(102), 60)),
    "deflate_shifted": ("deflate", lambda: layout_deflate(random.Random(103), 60, shifts=True)
                        + layout_malformed_deflate(random.Random(104), 60, shifts=True)),
    "deflate_large": ("deflate", lambda: layout_deflate(random.Random(105), 40, max_raw=4000)
                      + layout_deflate(random.Random(106), 40, max_raw=4000, shifts=True)
                      + layout_malformed_deflate(random.Random(107), 24) + layout_malformed_deflate(random.Random(108), 24, shifts=True)),
    "lz4_block": ("lz4_block", lambda: layout_lz4(random.Random(109), 40)),
    "bzip2": ("bzip2", lambda: layout_bzip2(random.Random(110), 24)),
    "lzma2": ("lzma2", lambda: layout_lzma2(random.Random(111), 24)),
    "lzma": ("lzma", lambda: layout_lzma(random.Random(112), 24)),
}
LZ4_DICTIONARY = textlike(4096, 36001)


def lz4_frame_independent(blocks_raw, bd=0x40, content_checksum=False, block_checksum=False):
    """B4 independent-block frame built by hand (FLG version 01, B.Indep=1)."""
    import oracle_xxh
    flg = 0x60 | (0x10 if block_checksum else 0) | (0x04 if content_checksum else 0)
    desc = bytes([flg, bd])
    out = bytearray(struct.pack("<I", 0x184D2204) + desc + bytes([(oracle_xxh.xxh32(desc) >> 8) & 0xFF]))
    for raw in blocks_raw:
        comp = lz4_block_compress(raw)
        if len(comp) >= len(raw):
            out += struct.pack("<I", len(raw) | 0x80000000) + raw
            blk = raw
        else:
            out += struct.pack("<I", len(comp)) + comp
            blk = comp
        if block_checksum:
            out += struct.pack("<I", oracle_xxh.xxh32(blk))
    out += struct.pack("<I", 0)
    if content_checksum:
        out += struct.pack("<I", oracle_xxh.xxh32(b"".join(blocks_raw)))
    return bytes(out)
