"""Inputs that pin down the edges of Deflate.compress (Deflate+Compress.swift:22-197): the 32 768 reach, the exact-key
table that records every visited position and no position inside a match, the 258 cap, 9-bit literals, the stored/static
choice, and units around the GPU link builder's tile size.  Shared by the CPU and GPU tests."""
import random

import helpers as H

TILE = 65536          # positions per link-builder tile (deflate_compress.cuh)


def _filler(rng, n):
    """compressible text without 0xFF bytes, so a 0xFF key never occurs in it and the block stays static Huffman"""
    t = H.textlike(n, rng.randint(0, 1 << 30))
    assert 0xFF not in t
    return t


def _no_repeat(rng, n, high):
    """n bytes with no repeated 3-byte key (all literals), exactly `high` of them >= 144 (9-bit literals)"""
    while True:
        b = [rng.randint(0, 143) for _ in range(n)]
        for p in rng.sample(range(n), high):
            b[p] = rng.randint(144, 255)
        keys = [bytes(b[i:i + 3]) for i in range(n - 2)]
        if len(set(keys)) == len(keys):
            return bytes(b)


def cases():
    rng = random.Random(1951)
    K = b"\xff\xff\xff\xfe"
    out = []
    # distance exactly 32 768 is a match, 32 769 is not (:166)
    out.append(("dist_32768", K + _filler(rng, 32768 - 4) + K + b"tail"))
    out.append(("dist_32769", K + _filler(rng, 32769 - 4) + K + b"tail"))
    # a too-far key is still recorded (:158): its second occurrence becomes the table entry for the third
    out.append(("far_then_near", K + _filler(rng, 40000) + K + _filler(rng, 100) + K + b"end"))
    # the nearest same-key position lies inside an earlier match (never recorded): the walk must pass it to reach a
    # visited one, near or far
    inner = b"ZABCDEFG"
    f1 = _filler(rng, 500)
    out.append(("hidden_in_match", inner + f1 + inner + _filler(rng, 300) + b"ABCD!"))
    out.append(("far_visited_near_unvisited", b"ABCxy" + _filler(rng, 30000) + inner + f1 + inner + _filler(rng, 200) + b"ABC?"))
    out.append(("visited_out_of_reach", b"ABCxy" + _filler(rng, 33000) + inner + f1 + inner + _filler(rng, 200) + b"ABC?"))
    # 258 caps and matches that run to the end
    out.append(("zeros_1000", bytes(1000)))
    out.append(("run_to_end", b"abc" * 400))
    out.append(("cap_then_short", b"q" + b"z" * 258 + b"q" + b"z" * 259 + b"q"))
    # 9-bit literals
    out.append(("high_literals", bytes(rng.randint(144, 255) for _ in range(3000))))
    # stored/static: 8 n + 10 + k bits with k 9-bit literals; k = 23 ties (stored), 22 does not (static)
    out.append(("tie_stored", _no_repeat(rng, 300, 23)))
    out.append(("tie_minus_one_static", _no_repeat(rng, 300, 22)))
    # the 65 535 bound is on n + 5: 65 530 incompressible bytes are stored, 65 531 are not
    rnd = bytes(rng.getrandbits(8) for _ in range(65531))
    out.append(("random_65530", rnd[:65530]))
    out.append(("random_65531", rnd))
    # around the tile size (keys live at positions 0 .. n - 3), and several tiles
    text = H.textlike(3 * TILE + 4000, 77)
    for d in (-1, 0, 1):
        out.append((f"tile{d:+d}", text[:TILE + 2 + d]))
    out.append(("three_tiles", text))
    out.append(("zeros_tiles", bytes(2 * TILE + 100)))
    out.append(("runs", b"".join(bytes([rng.randint(0, 3)]) * rng.randint(1, 600) for _ in range(400))))
    for n in range(0, 8):
        out.append((f"short_{n}", b"ab\x00ab\x00ab"[:n]))
    return out
