"""Inputs that pin down the edges of BZip2.compress (BZip2+Compress.swift:44-349): RLE1 runs around 4 and 255, block
boundaries, used-byte maps, periodic blocks whose rotations tie, zero runs around powers of two, last groups of 1 and 50
symbols and blocks that end with 1, 2 and 6 tables.  Each case is (name, data, block size).  Shared by the CPU and GPU
tests; the CPU test checks that each case exercises what its name says."""
import random

import helpers as H

RAW = 80000          # raw bytes per block per BlockSize step (BZip2+Compress.swift:47)


def cases():
    rng = random.Random(2026)
    text = H.textlike(300000, 77)
    out = [("empty", b"", 1), ("one_byte", b"a", 1)]
    for r in (3, 4, 5, 254, 255, 256, 259, 510):
        out.append((f"run_{r}", b"x" + b"a" * r + b"y", 1))
    out.append(("run_split_by_block", b"q" * (RAW - 2) + b"z" * 6, 1))
    for k in (1, 2, 3):
        for d in (-1, 0, 1):
            out.append((f"exact_blocks_k{k}_{d:+d}", text[: RAW * k + d], k))
    out.append(("two_blocks_k1", text[: 2 * RAW], 1))
    out.append(("rle_1_25x", b"".join(bytes([c]) * 4 for c in b"abcdefgh" * 100), 1))   # every run of 4 -> 5 bytes
    out.append(("one_used_byte", b"z" * 3, 1))
    out.append(("two_used_bytes", b"abba" * 50, 1))
    out.append(("all_256_bytes", bytes(range(256)), 1))
    out.append(("used_map_gaps", bytes([1, 17, 200, 17, 1, 255]) * 20, 1))
    out.append(("period_divides_n", b"abc" * 1000, 1))
    out.append(("period_not_dividing", b"abcd" * 1000 + b"ab", 1))
    out.append(("pointer_0", b"abcdefgh", 1))                 # rotation 0 is the smallest
    out.append(("pointer_last", b"zyxwvuts", 1))              # rotation 0 is the largest
    out.append(("issue_38", bytes([0, 1, 0, 1, 0, 0, 1, 0, 1]), 1))
    for s in (b"ban", b"banana", b"abracadabra", b"Hello, World!\n", b"bananas and more bananas"):
        out.append((f"string_{s[:8].decode().strip()}", s, 1))
    for k in (5, 6, 8):                                       # zero runs of 2^k - 1, 2^k, 2^k + 1 after MTF
        for d in (-1, 0, 1):                                  # BWT of (ab)^(L+1) is b^(L+1) a^(L+1): two runs of L
            out.append((f"zero_run_{(1 << k) + d}", b"ab" * ((1 << k) + d + 1), 1))
    # EOB lands as the first (last group of 1) or the 50th symbol of the last group
    out.append(("last_group_1", bytes(range(1, 50)) + bytes([0]), 1))
    out.append(("last_group_50", bytes(range(1, 49)) + bytes([0]), 1))
    out.append(("random_6_tables", bytes(rng.getrandbits(8) for _ in range(20000)), 1))
    out.append(("text_tables", text[:40000], 1))
    out.append(("mixed_selectors", text[:6000] + bytes(rng.getrandbits(8) for _ in range(6000)) + bytes(6000) + text[:6000], 1))
    out.append(("zeros_multi", bytes(250000), 2))
    out.append(("random_k9_short", bytes(rng.getrandbits(8) for _ in range(50000)), 9))
    return out
