"""Full-size BZip2.compress inputs for the rotation sort of bzip2_compress.cu (sort_kernel): blocks that need 15-17 prefix
doubling rounds (offsets h up to 2^19), blocks whose last round's keys span more than the block (2h > n), blocks whose
rotations tie in groups far larger than one warp's segment, RLE1 output that fills a block's scratch to rle_cap, 256 used
bytes with 6 tables and 14 400 selectors, and a unit whose three blocks need very different round counts.  Each case is
(name, data, block size); test_bzip2_compress_big_cpu.py checks that each reaches what its name says."""
import functools

import numpy as np

import helpers as H

RAW = 80000          # raw bytes per block per BlockSize step (BZip2+Compress.swift:47)

MANY_ROUNDS = ("fibonacci_k9", "thue_morse_k9", "cXdX_up_k9", "cXdX_down_k9", "X_X_k9", "period7_mutated_k9",
               "period1021_mutated_k9")
WIDE_KEYS = ("fibonacci_k5", "period7_mutated_k5", "period1021_mutated_k5")
TIES = ("abc_k9", "period7_cut_k9", "mississippi_k9")
EXPANSION = ("runs4_k9", "runs4_shifted_k1")
EXTREMES = ("random_k9", "mixed_selectors_k9")
MIXED = ("mixed_unit_k9",)


def no_run3(rng, n, lo=0, hi=256):
    """random bytes in [lo, hi) without three equal bytes in a row: RLE1 leaves them unchanged"""
    x = rng.integers(lo, hi, n, dtype=np.uint8)
    while True:
        bad = np.flatnonzero((x[2:] == x[1:-1]) & (x[1:-1] == x[:-2])) + 2
        if not len(bad):
            return x.tobytes()
        x[bad] = (x[bad].astype(np.int64) - lo + 1) % (hi - lo) + lo


def fibonacci(n):
    """the first n bytes of the Fibonacci word over 'ab' (no run of 3): rotations share prefixes of a third of n and more"""
    a, b = b"a", b"ab"
    while len(b) < n:
        a, b = b, b + a
    return b[:n]


def thue_morse(n):
    """the first n bytes of the Thue-Morse word over 'ab' (cube-free)"""
    t = np.zeros(1, dtype=np.uint8)
    while len(t) < n:
        t = np.concatenate([t, 1 - t])
    return (t[:n] + ord("a")).tobytes()


def bumped(x, d):
    """x with its last byte moved by d: x' sorts above x for d > 0 and below it for d < 0"""
    return x[:-1] + bytes([(x[-1] + d) % 256])


def dipped(x):
    """x' < x, differing in one byte near the middle and not in the last one"""
    q = len(x) // 2
    while x[q] < 2 or x[q] - 1 in (x[q - 1], x[q + 1]):
        q += 1
    return x[:q] + bytes([x[q] - 1]) + x[q + 1:]


def mutated_period(rng, p, n):
    """n bytes of period p with the last byte changed: rotations i and i + p agree for about n - p bytes"""
    u = no_run3(rng, p)
    s = bytearray((u * (n // p + 1))[:n])
    s[-1] = s[-1] ^ 0x40 if s[-1] ^ 0x40 != s[-2] else s[-1] ^ 0x41
    return bytes(s)


def runs_of_4(rng, runs):
    """`runs` runs of exactly 4 equal bytes, adjacent runs distinct: RLE1 writes 5 bytes per 4"""
    steps = rng.integers(1, 256, runs)                      # a non-zero step from each run's byte to the next
    return np.repeat((np.cumsum(steps) % 256).astype(np.uint8), 4).tobytes()


@functools.lru_cache(maxsize=None)
def cases():
    rng = np.random.default_rng(2027)
    n9, n5 = 9 * RAW, 5 * RAW
    X = no_run3(rng, n9 // 2 - 1)
    Y = no_run3(rng, n9 // 2)
    out = [
        # many rounds: 15-17 doubling rounds, h >= 2^16
        ("fibonacci_k9", fibonacci(n9), 9),
        ("thue_morse_k9", thue_morse(n9), 9),
        ("cXdX_up_k9", b"c" + X + b"d" + bumped(X, 1), 9),          # stopped early, the tie order is already right
        ("cXdX_down_k9", b"c" + X + b"d" + bumped(X, -1), 9),       # stopped early, 'c' and 'd' trade places
        ("X_X_k9", Y + dipped(Y), 9),                               # stopped early, only the pointer moves
        ("period7_mutated_k9", mutated_period(rng, 7, n9), 9),
        ("period1021_mutated_k9", mutated_period(rng, 1021, n9), 9),
        # the last round's (rank[i], rank[i + h mod n]) keys span 2h > n bytes
        ("fibonacci_k5", fibonacci(317811), 5),                     # the Fibonacci word of length F(28)
        ("period7_mutated_k5", mutated_period(rng, 7, n5), 5),
        ("period1021_mutated_k5", mutated_period(rng, 1021, n5), 5),
        # rotations that tie across the whole block, in groups of 60 000 and more
        ("abc_k9", b"abc" * (n9 // 3), 9),                          # the period divides n: rotation 0 ties
        ("period7_cut_k9", (b"abcdefg" * (n9 // 7 + 1))[:n9], 9),   # 7 does not divide n
        ("mississippi_k9", b"mississippi!" * (n9 // 12), 9),        # rotation 0 sorts sixth of 12: pointer 5 n / 12
        # RLE1 output at rle_cap: 900 000 bytes from 720 000, and the same runs cut by ten k = 1 block boundaries
        ("runs4_k9", runs_of_4(rng, n9 // 4), 9),
        ("runs4_shifted_k1", runs_of_4(rng, 10 * RAW // 4 + 1)[2:2 + 10 * RAW], 1),
        # 256 used bytes, 6 tables, 14 400 selectors; and regions that bring selector MTF index 5 late in the block
        ("random_k9", rng.integers(0, 256, n9, dtype=np.uint8).tobytes(), 9),
    ]
    # text, random bytes, four symbols, text: the greedy table choice comes back to its least recently used table (MTF
    # index 5) in the last quarter of the selectors (a property of these seeds, checked by the CPU test)
    text, sel = H.textlike(n9 // 2, 11), np.random.default_rng(102)
    out.append(("mixed_selectors_k9", text[:n9 // 4] + sel.integers(0, 256, n9 // 4, dtype=np.uint8).tobytes()
                + no_run3(sel, n9 // 4, 0, 4) + text[n9 // 4:], 9))
    # one unit, three blocks: 16 rounds, none (its 8-byte keys are already distinct), a single byte
    out.append(("mixed_unit_k9", thue_morse(n9) + rng.integers(0, 256, n9, dtype=np.uint8).tobytes() + b"x", 9))
    return tuple(out)


def by_name():
    return {name: (data, k) for name, data, k in cases()}
