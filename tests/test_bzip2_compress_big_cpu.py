"""The full-size cases of bzip2c_big_cases.py reach the rotation-sort edges their names claim.  A numpy model of sort_kernel
(bzip2_compress.cu) runs on each block's RLE1 bytes: 8-byte cyclic keys, then stable sorts of (rank[i], rank[i + h mod n])
keys with h = 8, 16, 32, ..., stopping after the first round that splits no group, ties left in index order as the stable
radix sort leaves them.  Its pointer must equal the one in the oracle's stream (DESIGN §4.11, lemma 1 at full size against
the oracle's SA-IS), and each near-miss variant of the model (a sort that stops early, a 16-bit offset, a rank sort that
skips its top digit, ties broken the other way) must change the BWT or the pointer of the cases listed against it.

A round with h >= n never runs once n > 8: before the round with offset h > 8 the partition is by the first h bytes, which
for h >= n is already the partition into equal rotations, so the round runs only if some rotations are equal (the block is
a power u^(n/p) of a primitive u) and the round h/2 still split a group.  Distinct rotations of u^(n/p) agree on at most
p - 1 <= n/2 - 1 bytes, so that last split came from h/2 < p, i.e. h < n.  The widest keys a full-size block reaches are
therefore those of a last round with n/2 < h < n, whose pairs span 2h > n bytes; the WIDE_KEYS cases get there.  Only
blocks of at most 8 RLE1 bytes with equal rotations, such as one_used_byte of bzip2c_cases.py, run a round with h >= n."""
import bz2

import numpy as np
import pytest

import bzip2c_big_cases as K
from test_bzip2_compress_cpu import bound

SORT_WARPS = 16          # sort_kernel's warps, each ranking one segment of the sorted keys


@pytest.fixture(scope="module")
def oc():
    import swco_bzip2c
    swco_bzip2c.lib()
    return swco_bzip2c


# ---- the model ----------------------------------------------------------------------------------------------------------
def rle1(block):
    """initialRle (BZip2+Compress.swift:265-283): runs of 4-255 become 4 bytes and a count"""
    a = np.frombuffer(block, dtype=np.uint8)
    if not len(a):
        return b""
    starts = np.flatnonzero(np.r_[True, a[1:] != a[:-1]])
    out = []
    for s, ln in zip(starts.tolist(), np.diff(np.r_[starts, len(a)]).tolist()):
        while ln > 0:
            r = min(ln, 255)
            out.append(a[s:s + 1].tobytes() * min(4, r) + (bytes([r - 4]) if r >= 4 else b""))
            ln -= r
    return b"".join(out)


def rle_cap(raw):
    """bzip2c::rle_cap: RLE1 writes at most 5 bytes per 4"""
    return raw + raw // 4


def blocks(data, k):
    return [data[at:at + K.RAW * k] for at in range(0, len(data), K.RAW * k)]


def segment(n):
    """the keys one warp of sort_kernel ranks (seg_bounds)"""
    return ((n + SORT_WARPS - 1) // SORT_WARPS + 31) // 32 * 32


def _rank(order, key, n):
    """rank[i] = the first sorted position whose key equals i's (rank_groups) -> (rank, groups, largest group)"""
    start = np.r_[True, key[1:] != key[:-1]]
    rank = np.empty(n, dtype=np.int64)
    rank[order] = np.maximum.accumulate(np.where(start, np.arange(n), 0))
    return rank, int(start.sum()), int(np.diff(np.r_[np.flatnonzero(start), n]).max())


def sort_model(r, max_rounds=None, h_bits=64, top_digit=True):
    """sort_kernel on the RLE1 bytes r -> dict(order, rank, rounds, hs, groups, largest).  The variants: stop after
    `max_rounds` rounds; keep h in `h_bits` bits; sort each rank half by its low 16 bits only (not `top_digit`)."""
    a = np.frombuffer(r, dtype=np.uint8).astype(np.uint64)
    n = len(a)
    idx = np.arange(n)
    key = np.zeros(n, dtype=np.uint64)
    for t in range(8):
        key = (key << np.uint64(8)) | a[(idx + t) % n]
    order = np.argsort(key, kind="stable")
    rank, groups, largest = _rank(order, key[order], n)
    hs, h = [], 8
    while groups < n and len(hs) < (max_rounds if max_rounds is not None else 64):
        hm = (h & ((1 << h_bits) - 1)) % n
        hi, lo = rank[order].astype(np.uint64), rank[(order + hm) % n].astype(np.uint64)
        full = hi * np.uint64(n) + lo
        m = np.uint64(0xFFFF)
        by = full if top_digit else ((hi & m) << np.uint64(16)) | (lo & m)
        p = np.argsort(by, kind="stable")
        order, full = order[p], full[p]
        rank, g2, _ = _rank(order, full, n)
        hs.append(h)
        if g2 == groups:
            break
        groups, h = g2, h * 2
    return dict(order=order, rank=rank, rounds=len(hs), hs=hs, groups=groups, largest=largest, n=n)


def bwt_and_pointer(r, order):
    """the emitted bytes B[(i - 1) mod n] and the pointer, rotation 0's place in the order"""
    a = np.frombuffer(r, dtype=np.uint8)
    return a[(order - 1) % len(a)].tobytes(), int(np.flatnonzero(order == 0)[0])


def symbols(bwt, used_low):
    """the number of MTF + RUNA/RUNB symbols mtfRle writes, EOB included: an MTF index is 0 exactly when the byte equals
    the one before it (at the start: the lowest used byte), and a zero run of L takes floor(log2(L + 1)) digits"""
    b = np.frombuffer(bwt, dtype=np.uint8)
    zero = b == np.r_[np.uint8(used_low), b[:-1]]
    edges = np.diff(np.r_[0, zero.astype(np.int8), 0])
    runs = np.flatnonzero(edges == -1) - np.flatnonzero(edges == 1)
    return int((~zero).sum()) + int(np.floor(np.log2(runs + 1)).sum()) + 1


def header(stream):
    """the first block header of a .bz2 stream -> dict(ptr, used, ntab, nsel, sel_mtf): fields at fixed offsets after the
    32-bit stream header, then one unary selector MTF index per group"""
    bits = np.unpackbits(np.frombuffer(stream[:200000], dtype=np.uint8))
    pos = 32

    def rd(k):
        nonlocal pos
        v = int(bits[pos:pos + k].dot(1 << np.arange(k - 1, -1, -1, dtype=np.int64)))
        pos += k
        return v

    assert rd(48) == 0x314159265359
    rd(32)
    assert rd(1) == 0
    ptr, maps = rd(24), rd(16)
    used = sum(bin(rd(16)).count("1") for j in range(16) if (maps >> (15 - j)) & 1)
    ntab, nsel = rd(3), rd(15)
    zeros = np.flatnonzero(bits[pos:pos + 6 * nsel] == 0)[:nsel]
    return dict(ptr=ptr, used=used, ntab=ntab, nsel=nsel, sel_mtf=np.diff(np.r_[-1, zeros]) - 1)


# ---- cached runs --------------------------------------------------------------------------------------------------------
_MODEL, _ORACLE = {}, {}


def model(name):
    """the model on every block of the case -> [(RLE1 bytes, raw length, model result)]"""
    if name not in _MODEL:
        data, k = K.by_name()[name]
        _MODEL[name] = [(rle1(b), len(b), sort_model(rle1(b))) for b in blocks(data, k)]
    return _MODEL[name]


def oracle_stream(oc, name):
    if name not in _ORACLE:
        data, k = K.by_name()[name]
        st, out, _ = oc.bzip2_compress(data, k)
        assert st == 0
        _ORACLE[name] = out
    return _ORACLE[name]


NAMES = [c[0] for c in K.cases()]


def test_families_cover_the_catalogue():
    fams = K.MANY_ROUNDS + K.WIDE_KEYS + K.TIES + K.EXPANSION + K.EXTREMES + K.MIXED
    assert sorted(fams) == sorted(NAMES) and len(set(NAMES)) == len(NAMES)


@pytest.mark.parametrize("name", NAMES)
def test_case_reaches_its_edge(name):
    res = model(name)
    for r, raw, m in res:
        print(f"{name}: raw {raw} n {m['n']} rounds {m['rounds']} last h {m['hs'][-1] if m['hs'] else '-'} "
              f"largest group {m['largest']} segment {segment(m['n'])}")
        if m["hs"] and m["n"] > 8:
            assert m["hs"][-1] < m["n"]                   # see the module docstring
    (r, raw, m), = res[:1]
    n, hs = m["n"], m["hs"]
    if name in K.MANY_ROUNDS:
        assert n == raw == 720000                         # no run of 4: RLE1 leaves the block unchanged
        assert m["rounds"] >= 15 and hs[-1] >= 1 << 17   # offsets past 2^16; h = 2^16 splits groups
    if name in K.WIDE_KEYS:
        assert n == raw and m["rounds"] >= 15 and 2 * hs[-1] > n
    if name in K.TIES:
        assert n == raw == 720000 and m["largest"] > segment(n)
    if name == "runs4_k9":
        assert n == rle_cap(raw) == 900000
    if name == "runs4_shifted_k1":                        # every block: 2 bytes of a cut run, 19 999 runs of 4, 2 bytes
        data, k = K.by_name()[name]
        for b in blocks(data, k):
            assert len(b) == 80000 and b[0] == b[1] != b[2] and b[-1] == b[-2] != b[-3]
        assert [m["n"] for _, _, m in res] == [2 + 5 * 19999 + 2] * 10
    if name == "mixed_unit_k9":
        assert [raw for _, raw, _ in res] == [720000, 720000, 1]
        rounds = [m["rounds"] for _, _, m in res]
        assert rounds[0] >= 15 and rounds[1] == 0 and rounds[2] == 0


def test_ties_are_whole_block_groups():
    c = {name: model(name)[0][2] for name in K.TIES}
    m = c["abc_k9"]
    assert m["groups"] == 3 and np.bincount(m["rank"]).max() == 240000 and m["rank"][0] == 0
    m = c["period7_cut_k9"]                                 # no two rotations equal, but 8-byte groups of ~100 000
    assert m["groups"] == m["n"] and m["largest"] > 100000 and m["rounds"] >= 15
    m = c["mississippi_k9"]
    assert m["groups"] == 12 and m["rank"][0] == 5 * 60000  # rotation 0 starts a group of 60 000 in the middle


@pytest.mark.parametrize("name", NAMES)
def test_oracle_header_matches_model(oc, name):
    r, raw, m = model(name)[0]
    h = header(oracle_stream(oc, name))
    bwt, ptr = bwt_and_pointer(r, m["order"])
    used = sorted(set(r))
    assert h["ptr"] == ptr == m["rank"][0]
    assert h["used"] == len(used)
    assert h["nsel"] == (symbols(bwt, used[0]) + 49) // 50
    assert 2 <= h["ntab"] <= 6
    if name in K.EXTREMES:
        assert h["used"] == 256 and h["ntab"] == 6
    if name == "random_k9":
        assert h["nsel"] == 14400
    if name == "mixed_selectors_k9":
        late = np.flatnonzero(h["sel_mtf"] == 5)
        assert len(late) and late[-1] > 3 * h["nsel"] // 4   # the least recently used table, in the last quarter


# each variant of sort_kernel and the cases that must tell it apart from the kernel
NEAR_MISSES = {
    "stop_after_4": (dict(max_rounds=4), ("fibonacci_k9", "thue_morse_k9", "cXdX_down_k9", "X_X_k9", "period7_mutated_k9",
                                         "period1021_mutated_k9", "fibonacci_k5", "mixed_unit_k9")),
    "h_16_bits": (dict(h_bits=16), ("fibonacci_k9", "period7_mutated_k9", "period1021_mutated_k5")),
    "no_top_digit": (dict(top_digit=False), ("X_X_k9", "fibonacci_k9", "runs4_k9")),
    "ties_descending": (None, ("abc_k9", "mississippi_k9")),
}


@pytest.mark.parametrize("variant", sorted(NEAR_MISSES))
def test_near_misses_are_caught(variant):
    kw, names = NEAR_MISSES[variant]
    for name in names:
        r, raw, m = model(name)[0]
        want = bwt_and_pointer(r, m["order"])
        if kw is None:                                    # the same partition, ties in descending index order
            got = bwt_and_pointer(r, np.lexsort((-np.arange(m["n"]), m["rank"])))
        else:
            got = bwt_and_pointer(r, sort_model(r, **kw)["order"])
        assert got != want, (variant, name)


def test_early_stop_moves_what_each_repeat_case_claims():
    """c X d X' with X' above X: the pairs an early stop leaves tied are already in order, so nothing moves; with X' below
    X the pair behind 'c' and 'd' swaps and the BWT changes.  X X' with X' below X in a middle byte: the pairs that swap,
    rotation 0's among them, have equal preceding bytes, so only the pointer moves"""
    for name, bwt_moves, ptr_moves in (("X_X_k9", False, True), ("cXdX_up_k9", False, False), ("cXdX_down_k9", True, False)):
        r, raw, m = model(name)[0]
        want = bwt_and_pointer(r, m["order"])
        got = bwt_and_pointer(r, sort_model(r, max_rounds=4)["order"])
        assert (got[0] != want[0], got[1] != want[1]) == (bwt_moves, ptr_moves), name


def test_model_equals_naive_sort():
    rng = np.random.default_rng(9)
    for t in range(400):
        n = int(rng.integers(1, 60))
        if t % 3 == 0:
            p = rng.integers(0, 3, int(rng.integers(1, 6)))
            s = np.resize(p, n).astype(np.uint8).tobytes()
        else:
            s = rng.integers(0, 2 + t % 4, n, dtype=np.uint8).tobytes()
        m = sort_model(s)
        rots = sorted(range(n), key=lambda j: (s[j:] + s[:j], j))
        assert bwt_and_pointer(s, m["order"]) == (bytes(s[j - 1] for j in rots), rots.index(0)), s
        assert m["rank"][0] == sum(s[j:] + s[:j] < s for j in range(n))
        if m["hs"] and m["hs"][-1] >= n:
            assert n <= 8, s


@pytest.mark.parametrize("name", NAMES)
def test_oracle_decodes_and_fits_bound(oc, name):
    import swco
    data, k = K.by_name()[name]
    out = oracle_stream(oc, name)
    assert bz2.decompress(out) == data
    assert len(out) <= bound(len(data), k)
    st, back = swco.bzip2_decompress(out)[:2]
    assert st == 0 and back == data
