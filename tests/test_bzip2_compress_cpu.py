"""The CPU restatement of BZip2.compress (oracle/bzip2_compress.c) against a line-by-line Python statement of
BZip2+Compress.swift, its SA-IS against a naive sort, the heap form of BZip2.lengths(from:) against the reference's
O(n^2) loop, and every stream back through Python's bz2 and the existing BZip2 restatement."""
import bz2
import heapq
import random
import shutil
import subprocess

import pytest

import bzip2c_cases as K

RUN_CAP = 255


@pytest.fixture(scope="module")
def oc():
    import swco_bzip2c
    swco_bzip2c.lib()
    return swco_bzip2c


# ---- the statement: BZip2+Compress.swift, BurrowsWheeler.swift, BZip2+Lengths.swift, Code.swift ----
class Bits:
    def __init__(self):
        self.bits = []

    def num(self, v, n):
        self.bits += [(v >> (n - 1 - k)) & 1 for k in range(n)]

    def data(self):
        b = self.bits + [0] * (-len(self.bits) % 8)
        return bytes(int("".join(map(str, b[i:i + 8])), 2) for i in range(0, len(b), 8))


def crc32_bzip2(data):
    c = 0xFFFFFFFF
    for v in data:
        c ^= v << 24
        for _ in range(8):
            c = ((c << 1) ^ 0x04C11DB7) & 0xFFFFFFFF if c & 0x80000000 else (c << 1) & 0xFFFFFFFF
    return c ^ 0xFFFFFFFF


def lengths_loop(stats, le_merge=True):
    """BZip2+Lengths.swift: the O(n^2) merge (<= picks the last index) and generateSizeTable's symbol order"""
    stats = list(stats)
    n = len(stats)
    cl, others = [0] * n, [-1] * n
    better = (lambda a, b: a <= b) if le_merge else (lambda a, b: a < b)
    while True:
        c1, m = -1, float("inf")
        for i in range(n):
            if stats[i] > 0 and better(stats[i], m):
                m, c1 = stats[i], i
        c2, m = -1, float("inf")
        for i in range(n):
            if stats[i] > 0 and better(stats[i], m) and i != c1:
                m, c2 = stats[i], i
        if c2 < 0:
            break
        stats[c1] += stats[c2]
        stats[c2] = 0
        cl[c1] += 1
        while others[c1] >= 0:
            c1 = others[c1]
            cl[c1] += 1
        others[c1] = c2
        cl[c2] += 1
        while others[c2] >= 0:
            c2 = others[c2]
            cl[c2] += 1
    return cl


def lengths_heap(stats):
    """the engine's form: a heap keyed (frequency ascending, symbol descending); merged weight stays under c1"""
    h = [(f, -i) for i, f in enumerate(stats)]
    heapq.heapify(h)
    cl, members = [0] * len(stats), {i: [i] for i in range(len(stats))}
    while len(h) > 1:
        f1, c1 = heapq.heappop(h)
        f2, c2 = heapq.heappop(h)
        c1, c2 = -c1, -c2
        for s in members[c1] + members[c2]:
            cl[s] += 1
        members[c1] += members.pop(c2)
        heapq.heappush(h, (f1 + f2, -c1))
    return cl


def statement(data, k=1, trace=None, variant=None):
    """BZip2.compress(data:blockSize:) line by line; `variant` names a near miss that each catalogue edge must catch"""
    tr = trace if trace is not None else {}
    w = Bits()
    w.num(0x425A, 16); w.num(0x68, 8); w.num(0x30 + k, 8)
    raw = k * 100 * 800
    total = 0
    for i in range(0, len(data), raw):
        block = data[i:i + raw]
        c = crc32_bzip2(block)
        total = (((total << 1) | (total >> 31)) & 0xFFFFFFFF) ^ c
        w.bits += [int(b) for b in "001100010100000101011001001001100101001101011001"]
        w.num(c, 32)
        _process(block, w, tr, variant)
    w.bits += [int(b) for b in "000101110111001001000101001110000101000010010000"]
    w.num(total, 32)
    return w.data()


def _process(block, w, tr, variant):
    cap = 256 if variant == "run_cap_256" else RUN_CAP
    out, i = [], 0
    while i < len(block):
        r = 1
        while i + 1 < len(block) and block[i] == block[i + 1] and r < cap:
            r += 1
            i += 1
        out += [block[i]] * min(4, r) + ([r - 4] if r >= 4 else [])
        tr.setdefault("runs", set()).add(r)
        i += 1
    tr.setdefault("rle_ratio", []).append(len(out) / max(1, len(block)))
    n = len(out)
    rots = sorted(range(n), key=lambda j: out[j:] + out[:j])
    bwt = [out[j - 1] for j in rots]
    r0 = out
    ptr = sum(1 for j in range(n) if (out[j:] + out[:j] <= r0 if variant == "pointer_le" else out[j:] + out[:j] < r0))
    tr.setdefault("pointer", []).append((ptr, n))
    used = sorted(set(bwt))
    tr.setdefault("used", []).append(len(used))
    d, syms, z, maxsym = list(used), [], 0, 1
    for j, c in enumerate(bwt):
        idx = d.index(c)
        if idx == 0:
            z += 1
        if (idx == 0 and j == n - 1) or idx != 0:
            if z:
                tr.setdefault("zruns", set()).add(z)
            while z > 0:
                q = (z + 1) // 2 - 1
                syms.append(0 if z - 2 * q == 1 else 1)
                z = q
        if idx:
            syms.append(idx + 1)
            maxsym = max(maxsym, idx + 1)
        d.insert(0, d.pop(idx))
    syms.append(maxsym + 1)
    A = maxsym + 2
    tr.setdefault("last_group", []).append((len(syms) - 1) % 50 + 1)
    tables, sels, ties = [], [], 0
    for g in range(0, len(syms), 50):
        stats = [1] * A
        for s in syms[g:g + 50]:
            stats[s] += 1
        scores = [sum(f * t[s] for s, f in enumerate(stats)) for t in tables]
        best = min(scores) if scores else float("inf")
        ties += scores.count(best) > 1            # two tables share the least score: the first one wins
        pick = (len(scores) - 1 - scores[::-1].index(best)) if (variant == "choice_le" and scores) else \
            (scores.index(best) if scores else -1)
        if len(tables) == 6:
            sels.append(pick)
            continue
        cl = lengths_loop(stats, le_merge=variant != "merge_lt")
        counts = sorted(cl)
        if variant == "lengths_by_frequency":
            cand = list(cl)
        else:
            cand = counts                     # generateSizeTable: lengths in increasing order to symbols 0, 1, 2, ...
        cs = sum(f * l for f, l in zip(stats, cand))
        if cs < best:
            tables.append(cand)
            sels.append(len(tables) - 1)
        else:
            sels.append(pick)
    tr.setdefault("tables", []).append(len(tables))
    tr["ties"] = tr.get("ties", 0) + ties
    if len(tables) == 1 and variant != "no_duplicate":
        tables.append(tables[0])
    w.num(0, 1); w.num(ptr, 24)
    maps = [int(any(c // 16 == m for c in used)) for m in range(16)]
    w.bits += maps
    for m in range(16):
        if maps[m]:
            w.bits += [int(m * 16 + j in used) for j in range(16)]
    w.num(len(tables), 3); w.num(len(sels), 15)
    order = list(range(len(tables)))
    for s in sels:
        idx = order.index(s)
        tr.setdefault("sel_mtf", set()).add(idx)
        w.bits += [1] * idx + [0]
        order.insert(0, order.pop(idx))
    for t in tables:
        prev = t[0]
        w.num(prev, 5)
        for l in t:
            w.bits += [1, 1] * (prev - l) if prev > l else [1, 0] * (l - prev)
            prev = l
            w.bits.append(0)
    codes = []
    for t in tables:                          # Code.huffmanCodes: canonical in (length, symbol) order, MSB first
        code, lb, cd = -1, None, {}
        for s in sorted(range(A), key=lambda s: (t[s], s)):
            code += 1
            if lb is not None and t[s] != lb:
                code <<= t[s] - lb
            if lb is None:
                code = 0
            lb = t[s]
            cd[s] = code
        codes.append(cd)
    for j, s in enumerate(syms):
        t = sels[j // 50]
        w.num(codes[t][s], tables[t][s])


def bound(n, k):
    raw, bits = 80000 * k, 112
    for at in range(0, n, raw):
        r = min(raw, n - at)
        R = r + r // 4
        bits += 395 + 6 * ((R + 50) // 50) + 6 * 283 + 11 * (R + 1)
    return (bits + 7) // 8


SMALL = [c for c in K.cases() if len(c[1]) <= 4100]


@pytest.mark.parametrize("name,data,k", SMALL, ids=[c[0] for c in SMALL])
def test_statement_equals_oracle(oc, name, data, k):
    assert statement(data, k) == oc.bzip2_compress(data, k)[1]


@pytest.mark.parametrize("name,data,k", K.cases(), ids=[c[0] for c in K.cases()])
def test_oracle_decodes_and_fits_bound(oc, name, data, k):
    import swco
    st, out, _ = oc.bzip2_compress(data, k)
    assert st == 0 and bz2.decompress(out) == data
    assert len(out) <= bound(len(data), k)
    ost, back = swco.bzip2_decompress(out)[:2]
    assert ost == 0 and back == data
    if shutil.which("bzip2"):                       # libbz2's own command-line decoder, where the system has it
        assert subprocess.run(["bzip2", "-dc"], input=out, capture_output=True, check=True).stdout == data


def test_catalogue_exercises_its_edges():
    tr = {}
    for name, data, k in SMALL:
        statement(data, k, tr)
    assert {3, 4, 5, 254, 255}.issubset(tr["runs"])
    assert 1.25 in tr["rle_ratio"]
    assert {1, 2, 256}.issubset(set(tr["used"]))
    assert any(p == 0 for p, n in tr["pointer"]) and any(p == n - 1 and n > 1 for p, n in tr["pointer"])
    assert {31, 32, 33, 63, 64, 65, 255, 256, 257}.issubset(tr["zruns"])
    assert {1, 50}.issubset(set(tr["last_group"]))
    assert {1, 2}.issubset(set(tr["tables"]))
    big = {}
    for name, data, k in K.cases():
        if name in ("random_6_tables", "mixed_selectors", "text_tables"):
            statement(data, k, big)
    assert 6 in big["tables"] and set(range(6)).issubset(big["sel_mtf"])
    assert big["ties"] > 0                          # two tables score the same: the first one wins


def raw_blocks_and_runs(data, k):
    """the raw blocks of compress(data:blockSize:) (:49-51) and the RLE1 run lengths of each"""
    raw, out = 80000 * k, []
    for at in range(0, len(data), raw):
        block, runs, i = data[at:at + raw], [], 0
        while i < len(block):
            r = 1
            while i + r < len(block) and block[i + r] == block[i] and r < RUN_CAP:
                r += 1
            runs.append(r)
            i += r
        out.append((len(block), runs))
    return out


def test_block_cases_exercise_their_edges():
    c = {name: (data, k) for name, data, k in K.cases()}
    b = raw_blocks_and_runs(*c["run_split_by_block"])
    assert len(b) == 2 and b[0][1][-1] == 2 and b[1][1][0] == 4            # a run of 6 cut into 2 + 4 by the boundary
    for k in (1, 2, 3):
        for d, sizes in ((-1, [80000 * k - 1]), (0, [80000 * k]), (1, [80000 * k, 1])):
            assert [n for n, _ in raw_blocks_and_runs(*c[f"exact_blocks_k{k}_{d:+d}"])] == sizes
    assert [n for n, _ in raw_blocks_and_runs(*c["two_blocks_k1"])] == [80000, 80000]
    assert [n for n, _ in raw_blocks_and_runs(*c["zeros_multi"])] == [160000, 90000]
    assert len(c["period_not_dividing"][0]) % 4 and not len(c["period_divides_n"][0]) % 3
    assert len(set(c["all_256_bytes"][0])) == 256


@pytest.mark.parametrize("variant", ["lengths_by_frequency", "merge_lt", "choice_le", "run_cap_256", "pointer_le",
                                     "no_duplicate"])
def test_near_misses_are_caught(oc, variant):
    cases = list(SMALL) + [c for c in K.cases() if c[0] in ("random_6_tables",)]
    assert any(statement(d, k, variant=variant) != oc.bzip2_compress(d, k)[1] for _, d, k in cases), variant


def test_suffix_array_as_written_equals_naive(oc):
    rng = random.Random(5)
    for t in range(3000):
        n = rng.randint(0, 40)
        if t % 3 == 0:
            p = [rng.randint(0, 3) for _ in range(rng.randint(1, 5))]
            s = (p * (n // len(p) + 1))[:n]
        else:
            s = [rng.randint(0, 2 + t % 5) for _ in range(n)]
        d = s + s                                   # BurrowsWheeler.transform sorts the doubled string
        assert oc.suffix_array(d, 8) == sorted(range(len(d) + 1), key=lambda i: d[i:]), s


def test_rotation_property(oc):
    """sorting rotations with any tie order gives the BWT of the doubled-string suffix array, and the pointer is the
    number of rotations strictly below rotation 0"""
    rng = random.Random(6)
    for t in range(1500):
        n = rng.randint(1, 30)
        p = [rng.randint(0, 2) for _ in range(rng.randint(1, 4))]
        s = (p * n)[:n] if t % 2 else [rng.randint(0, 2) for _ in range(n)]
        sa = oc.suffix_array(s + s, 4)
        bwt, ptr = [], 0
        for x in sa[1:]:
            if x < n:
                bwt.append(s[x - 1] if x > 0 else s[-1])
            elif x == n:
                ptr = len(bwt)
        rots = sorted(range(n), key=lambda j: (s[j:] + s[:j], rng.random()))
        assert bwt == [s[j - 1] for j in rots]
        assert ptr == sum(1 for j in range(n) if s[j:] + s[:j] < s)


def test_heap_build_equals_reference_loop(oc):
    rng = random.Random(7)
    for t in range(4000):
        A = rng.randint(3, 258)
        stats = [1] * A
        for _ in range(rng.randint(1, 50)):
            stats[min(A - 1, int(rng.expovariate(0.3 + t % 5)))] += 1
        loop = lengths_loop(stats)
        assert lengths_heap(stats) == loop
        assert max(loop) <= 11                      # lemma 4: a group weighs at most 308 < F(14) = 377
        if t % 40 == 0:
            assert oc.lengths(stats) == sorted(loop)


def test_adversarial_bound(oc):
    rng = random.Random(8)
    for data, k in [(bytes(rng.getrandbits(8) for _ in range(100000)), 1),
                    (b"".join(bytes([c]) * 4 for c in bytes(rng.getrandbits(8) for _ in range(25000))), 1),
                    (bytes(range(256)) * 400, 1)]:
        st, out, _ = oc.bzip2_compress(data, k)
        assert st == 0 and len(out) <= bound(len(data), k)


def test_invalid_block_size(oc):
    for k in (0, 10):
        assert oc.bzip2_compress(b"abc", k)[0] == 4
