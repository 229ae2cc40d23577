"""Inputs for the LZ4 compressor tests (LZ4+Compress.swift), shared by the CPU and the GPU test files.

`py_block` is a plain-Python statement of compress(block:_:) (:156-298).  Its `variant` switch builds the near-misses a
wrong implementation would produce, so every edge case below can prove that it tells them apart from the reference."""
import json
import os
import random

# fixtures of the compress side (tests/golden/manifest_compress.json): the dictionary of the reference's small-dictionary test
with open(os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "manifest_compress.json")) as _f:
    COMPRESS_MANIFEST = json.load(_f)

STRINGS = [b"ban", b"banana", b"abaaba", b"abracadabra", b"cabbage", b"baabaabac", b"AAAAAAABBBBCCCD", b"AAAAAAA",
           b"qwertyuiopasdfghjklzxcvbnmQWERTYUIOPASDFGHJKLZXCVBNM1234567890", bytes(range(256))]   # LZ4CompressionTests.swift:29-48
TRICKY = bytes([0x61, 0x6C, 0x20, 0x2D, 0x43, 0x20, 0x2D, 0x43, 0x20, 0x2D, 0x2D, 0x01, 0x02, 0x03, 0x04, 0x05, 0x06, 0x07,
                0x08, 0x09, 0x00])                                                                   # :162-171
TRICKY_OPTS = dict(independentBlocks=False, blockChecksums=True, contentChecksum=True, contentSize=True)


def _len_bytes(rest):
    out = bytearray()
    while rest >= 0:
        out.append(min(rest, 255))
        rest -= 255
    return bytes(out)


def py_block(block, dictionary=b"", variant=None):
    """compress(block:_:).  variant: None = the reference; "record_all" also records positions inside matches (a naive
    latest-occurrence table); "dict_tail" also records the last 4 dictionary positions; "far" accepts distance 65 536,
    "near" refuses 65 535."""
    b = bytes(dictionary) + bytes(block)
    end = len(b)
    table = {}
    dict_end = len(dictionary) - (0 if variant == "dict_tail" else 4)
    for i in range(0, max(dict_end, 0)):
        if i + 4 <= end:
            table[b[i:i + 4]] = i
    i = len(dictionary)
    lit_start = i
    out = bytearray()
    limit = {"far": 65536, "near": 65534}.get(variant, 65535)
    while i < end - 9:
        key = b[i:i + 4]
        q = table.get(key)
        table[key] = i
        if q is None or i - q > limit:
            i += 1
            continue
        n = 4
        while i + n < end - 5 and b[i + n] == b[q + n]:
            n += 1
        if end - i < 12:
            break
        lit = i - lit_start
        out.append(min(15, lit) << 4 | min(15, n - 4))
        out += _len_bytes(lit - 15) + b[lit_start:i]
        out += bytes([(i - q) & 0xFF, ((i - q) >> 8) & 0xFF])
        if variant == "record_all":
            for k in range(i + 1, i + n):
                if k < end - 9:
                    table[b[k:k + 4]] = k
        i += n
        out += _len_bytes(n - 19)
        lit_start = i
    lit = end - lit_start
    out.append(min(15, lit) << 4)
    out += _len_bytes(lit - 15) + b[lit_start:]
    return bytes(out)


def _rand(rng, n):
    return bytes(rng.getrandbits(8) for _ in range(n))


def _distinct(rng, n, avoid=()):
    """n random bytes whose 4-byte keys do not repeat (rejection on the running key set)"""
    out = bytearray(_rand(rng, 3))
    keys = set(avoid)
    while len(out) < n:
        c = rng.getrandbits(8)
        k = bytes(out[-3:]) + bytes([c])
        if k in keys:
            continue
        keys.add(k)
        out.append(c)
    return bytes(out)


def edge_blocks():
    """(name, block, dictionary, variant it must differ from or None) — raw-block edge cases"""
    rng = random.Random(20261015)
    cases = []
    for n in range(0, 17):                                     # around the 5 / 9 / 11 / 12 bounds
        cases.append((f"same{n}", b"a" * n, b"", None))
        cases.append((f"ab{n}", (b"abcd" * 5)[:n], b"", None))
    for n in (10, 11, 12, 13, 14):                             # a 4-byte match that starts exactly at the last legal position
        cases.append((f"tailmatch{n}", b"wxyz" + bytes(range(100, 100 + n - 8)) + b"wxyz", b"", None))
    # a key at distance 65 535 matches, at 65 536 it does not
    key = b"\xAA\xBB\xCC\xDD"
    for dist, var in ((65535, "near"), (65536, "far")):
        filler = _distinct(rng, dist - 4, avoid={key})
        cases.append((f"dist{dist}", key + filler + key + b"\x01\x02\x03\x04\x05\x06\x07\x08\x09\x0a\x0b\x0c", b"",
                      var))
    # literal runs and match lengths at the token / extension-byte edges
    for v in (15, 19, 15 + 255, 19 + 255, 15 + 510, 19 + 510, 14, 18, 270, 274):
        lits = _distinct(rng, v)
        cases.append((f"lit{v}", lits + lits[:8] + _distinct(rng, 16), b"", None))
        src = _distinct(rng, 8)
        cases.append((f"match{v}", src + (src * (v // 8 + 2))[:v] + _distinct(rng, 16), b"", None))
    # a match source inside an earlier match: the reference never recorded those positions
    p = _distinct(rng, 20)
    cases.append(("inside_match", p + p + p[5:13] + _distinct(rng, 20, avoid={p[k:k + 4] for k in range(17)}), b"",
                  "record_all"))
    # keys in the last 4 dictionary bytes are never candidates
    d = _distinct(rng, 60)
    cases.append(("dict_tail", d[-4:] + d[-3:] + _distinct(rng, 24, avoid={d[k:k + 4] for k in range(57)}), d, "dict_tail"))
    cases.append(("dict4", b"abcdabcd" + b"0123456789abcdef", b"abcd", None))
    big = _rand(rng, 70000)
    cases.append(("dict_big", big[-3000:-1000] + _rand(rng, 5000) + big[100:2000], big, None))
    return cases


def compressible_equal_size(max_tries=4000):
    """a block whose compressed form is exactly as long as the block (it must stay compressed: :112 is a strict >)"""
    rng = random.Random(7)
    for _ in range(max_tries):
        n = rng.randint(40, 400)
        data = bytearray(_rand(rng, n))
        k, at, src = rng.randint(4, 12), rng.randint(20, n - 20), rng.randint(0, 10)
        data[at:at + k] = data[src:src + k]
        data = bytes(data)
        if len(py_block(data)) == len(data):
            return data
    raise AssertionError("no equal-size block found")


def frame_inputs():
    """(name, data) pairs for the option sweep"""
    rng = random.Random(99)
    words = [bytes(rng.choice(b"etaoinshrdlu ") for _ in range(rng.randint(2, 9))) for _ in range(300)]
    text = b" ".join(rng.choice(words) for _ in range(30000))[:150000]
    return [("empty", b""), ("text", text), ("random", _rand(rng, 70001)), ("zeros", bytes(200000)),
            ("mixed", text[:40000] + bytes(30000) + _rand(rng, 9000) + text[:20000])]


SWEEP_BLOCK_SIZES = (1024, 65536, 77777, 4 << 20)
