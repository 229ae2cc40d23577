"""Inputs aimed at the GPU machinery that replaces the reference compressors' hash tables, and a small model of it.

Deflate (csrc/deflate_compress.cu): link_kernel gives one warp to each tile [65 536 t, 65 536 (t + 1)) of key positions
and threads the REACH = 32 768 positions in front of it (the halo) and the tile onto 4096 hash-bucket chains, 32
positions per warp step counted from the window start r0 = max(0, t0 - REACH).  A key is d[p] | d[p+1] << 8 |
d[p+2] << 16; x = key * 0x9E3779B1 mod 2^24 is split into the bucket x >> 12 and the tag x & 0xFFF, and link[p] is the
first entry down the bucket chain with p's tag.  parse_kernel walks link[] to the first visited position and drops a
checkpoint at the first symbol at or after every CHUNK = 4096 input bytes (mark()); emit_kernel places each chunk's
symbols from its checkpoint's bit count, and seam_kernel merges the words two chunks share.

LZ4 (csrc/lz4_compress.cu): lz4c_chain_kernel gives one warp to a unit's whole window (dictionary + block).  The key is
the 4 bytes at p big-endian, its bucket (key * 2654435761 mod 2^32) >> 20.  A forward pass links every position to the
nearest earlier one of its bucket (at most 65 535 back); a backward pass, 32 positions at a time from the end, rewrites
each link in place to the first position down the bucket chain with an equal key.

`deflate_model` / `lz4_model` restate that machinery position by position.  Their `variant` switch builds near misses of
it ("halo_short": the halo one position short; "bucket": bucket equality in place of key equality; "late_checkpoint": a
checkpoint's bit count taken one symbol late; "write_first": the backward pass writing a link before the other lanes of
its step have read theirs; "front_to_back": the backward pass going from the front).  Every case below names the edges
it is built to reach as tuples, and `deflate_edge` / `lz4_edge` check them on the model."""
import functools
import random

import numpy as np

import deflate_writer as W
import helpers as H

TILE, REACH, CHUNK = 65536, 32768, 4096          # deflate_compress.cuh
MAX_UNIT = 1 << 32
L_REACH, MAX_BLOCK, MAX_DICT = 65535, 4 << 20, 64 << 10   # lz4_compress.cu / lz4_compress.cuh
STEP = 32                                       # positions per warp step of both link builders

# bytes that neither H.textlike's filler nor the keys below (all bytes >= 0x80) use: one in front of a destination key
# keeps the filler in front of it from starting a match that would swallow the key
GUARDS = bytes(b for b in range(1, 0x80) if b not in H.textlike(1 << 16, 0))


# ---- keying ------------------------------------------------------------------------------------------------------------

def d_key(b, p):
    return b[p] | b[p + 1] << 8 | b[p + 2] << 16


def d_mix(key):
    """-> (bucket, tag) of a 3-byte Deflate key"""
    x = (key * 0x9E3779B1) & 0xFFFFFF
    return x >> 12, x & 0xFFF


def l_key(b, p):
    return int.from_bytes(bytes(b[p:p + 4]), "big")


def l_bucket(key):
    return ((key * 2654435761) & 0xFFFFFFFF) >> 20


@functools.lru_cache(maxsize=None)
def _d_high_keys_by_bucket():
    """all 2^24 Deflate keys, brute force: bucket -> the keys of that bucket whose three bytes are >= 0x80"""
    k = np.arange(1 << 24, dtype=np.uint64)
    k = k[(k & np.uint64(0x808080)) == np.uint64(0x808080)]
    b = ((k * np.uint64(0x9E3779B1)) & np.uint64(0xFFFFFF)) >> np.uint64(12)
    order = np.argsort(b, kind="stable")
    k, b = k[order], b[order]
    cuts = np.searchsorted(b, np.arange(4097))
    return [k[cuts[i]:cuts[i + 1]] for i in range(4096)]


def d_bucket_keys(rng, bucket, m):
    """m different 3-byte keys (as bytes) of one Deflate bucket, every byte >= 0x80"""
    ks = _d_high_keys_by_bucket()[bucket]
    return [int(k).to_bytes(3, "little") for k in rng.sample(list(ks), m)]


@functools.lru_cache(maxsize=None)
def _l_groups():
    """birthday grouping of random 4-byte LZ4 keys with every byte >= 0x80: buckets that got at least 8 of them"""
    rng = np.random.default_rng(4096)
    keys = np.unique(rng.integers(0, 1 << 32, size=1 << 17, dtype=np.uint64) | np.uint64(0x80808080))
    bk = ((keys * np.uint64(2654435761)) & np.uint64(0xFFFFFFFF)) >> np.uint64(20)
    groups = {}
    for k, b in zip(keys.tolist(), bk.tolist()):
        groups.setdefault(b, []).append(k)
    return {b: g for b, g in groups.items() if len(g) >= 8}


def l_bucket_keys(rng, m, avoid=()):
    """m different 4-byte keys (as bytes) of one LZ4 bucket not in `avoid`, every byte >= 0x80"""
    groups = _l_groups()
    b = rng.choice(sorted(set(groups) - set(avoid)))
    return b, [k.to_bytes(4, "big") for k in rng.sample(groups[b], m)]


def high(rng, n):
    return bytes(rng.randint(0x80, 0xFF) for _ in range(n))


class Layout:
    """filler text with byte strings placed at chosen positions; `dest` puts a fresh guard byte in front"""

    def __init__(self, n, seed):
        self.b = bytearray(H.textlike(n, seed))
        self.g = 0

    def put(self, p, s):
        self.b[p:p + len(s)] = s
        return p

    def dest(self, p, s):
        assert self.g < len(GUARDS), "more destinations than guard bytes"
        self.b[p - 1] = GUARDS[self.g]
        self.g += 1
        return self.put(p, s)

    def data(self):
        return bytes(self.b)


def distinct_run(rng, n, high_at=(), seen=None):
    """n bytes whose 3-byte keys never repeat (so a parse takes them all as literals); bytes at `high_at` are >= 144
    (9-bit literals), the others are < 144 and outside the filler's alphabet"""
    low = [b for b in range(0, 144) if b in GUARDS or b >= 0x80]
    hi = list(range(144, 256))
    seen = set() if seen is None else seen
    high_at = set(high_at)
    while True:
        out = bytearray()
        for i in range(n):
            pool = hi if i in high_at else low
            for _ in range(200):
                c = rng.choice(pool)
                if i < 2 or (out[-2], out[-1], c) not in seen:
                    break
            else:
                break
            if i >= 2:
                seen.add((out[-2], out[-1], c))
            out.append(c)
        if len(out) == n:
            return bytes(out)


# ---- Deflate model -----------------------------------------------------------------------------------------------------

def d_links(b, variant=None):
    """link[p] of link_kernel: the nearest earlier position with p's key (or, for "bucket", p's bucket) within REACH and
    inside the window of p's tile"""
    nk = max(len(b) - 2, 0)
    link, last = [0] * nk, {}
    for p in range(nk):
        k = d_key(b, p)
        t0 = p - p % TILE
        r0 = max(0, t0 - REACH + (1 if variant == "halo_short" and t0 else 0))
        h = d_mix(k)[0] if variant == "bucket" else k
        q = last.get(h)
        if q is not None and q >= r0 and p - q <= REACH:
            link[p] = p - q
        last[h] = p
    return link


def _d_bits(b, pos, ln, dist):
    if ln == 0:
        return 8 if b[pos] < 144 else 9
    ls, _ = W.len_symbol(ln)
    ds, _ = W.dist_symbol(dist)
    return (7 if ls <= 279 else 8) + W.LEN_EXTRA[ls - 257] + 5 + W.DIST_EXTRA[ds]


class DeflateModel:
    """parse_kernel over link[]: symbols (position, length, distance; length 0 for a literal), their first bits, the
    checkpoints [(symbol index, bit)] of every chunk, the stream's bit count and its bytes"""

    def __init__(self, data, variant=None):
        b = self.b = bytes(data)
        n = self.n = len(b)
        self.link = link = d_links(b, variant)
        vis = self.vis = bytearray(max(n - 2, 0))
        syms, i = [], 0
        while i + 2 < n:
            q, dd, found = i, link[i], False
            while dd:
                q -= dd
                if i - q > REACH:
                    break
                if vis[q]:
                    found = True
                    break
                dd = link[q]
            vis[i] = 1
            if not found:
                syms.append((i, 0, 0))
                i += 1
                continue
            ln = 3
            while i + ln < n and ln < 258 and b[i + ln] == b[q + ln]:
                ln += 1
            syms.append((i, ln, i - q))
            i += ln
        syms += [(p, 0, 0) for p in range(i, n)]
        self.syms = syms
        self.at = {s[0]: k for k, s in enumerate(syms)}
        self.first_bit, bit = [], 3
        for s in syms:
            self.first_bit.append(bit)
            bit += _d_bits(b, *s)
        self.sym_end = bit
        self.bits = bit + 7
        self.nch = (n + CHUNK - 1) // CHUNK if n else 1
        self.cp = [(0, 3)]
        k = 0
        for c in range(1, self.nch):
            while k < len(syms) and syms[k][0] < c * CHUNK:
                k += 1
            late = variant == "late_checkpoint" and k < len(syms)
            self.cp.append((k, self.first_bit[k] + (_d_bits(b, *syms[k]) if late else 0) if k < len(syms) else self.sym_end))
        self.stored = n + 5 <= (self.bits + 7) // 8 and n + 5 <= 65535
        self.out = self._emit()

    def _emit(self):
        n, b = self.n, self.b
        if self.stored:
            return bytes([1, n & 0xFF, n >> 8, (n ^ 0xFFFF) & 0xFF, (n ^ 0xFFFF) >> 8]) + b
        w = W.DeflateWriter()
        toks, run = [], bytearray()
        for p, ln, dist in self.syms:
            if ln == 0:
                run.append(b[p])
                continue
            if run:
                toks.append(bytes(run))
                run = bytearray()
            toks.append(W.Match(ln, dist))
        if run:
            toks.append(bytes(run))
        w.fixed(toks, final=True)
        stream, nbits = w.finish()
        assert nbits == self.bits
        # each chunk places its symbols from its checkpoint's bit count (the last one also places end-of-block)
        v = int.from_bytes(stream, "little")
        true_start = [0] + [self.first_bit[k] if k < len(self.syms) else self.sym_end for k, _ in self.cp[1:]]
        out = 0
        for c in range(self.nch):
            s0 = true_start[c]
            s1 = true_start[c + 1] if c + 1 < self.nch else self.bits
            seg = (v >> s0) & ((1 << (s1 - s0)) - 1)
            out |= seg << (self.cp[c][1] if c else 0)
        size = (self.bits + 7) // 8
        return (out & ((1 << (8 * size)) - 1)).to_bytes(size, "little")

    def sym(self, p):
        k = self.at.get(p)
        return None if k is None else self.syms[k]

    def chunk_syms(self, c):
        k0 = self.cp[c][0]
        k1 = self.cp[c + 1][0] if c + 1 < self.nch else len(self.syms)
        return self.syms[k0:k1]


def deflate_model(data, variant=None):
    return DeflateModel(data, variant).out


def _window_start(t):
    return max(0, t * TILE - REACH)


def deflate_edge(m, e):
    """True when the model reaches edge `e`"""
    kind, a = e[0], e[1:]
    b = m.b
    if kind == "match":                       # a match starts at p with distance dist
        s = m.sym(a[0])
        return s is not None and s[1] > 0 and s[2] == a[1]
    if kind == "literal":
        s = m.sym(a[0])
        return s is not None and s[1] == 0
    if kind == "halo":                        # q lies in the halo of tile t, at lane x of its warp step
        q, t, x = a
        return t >= 1 and t * TILE - REACH <= q < t * TILE and (q - _window_start(t)) % STEP == x % STEP
    if kind == "tile":                        # p lies in tile t, at lane x of its warp step
        p, t, x = a
        return p // TILE == t and (p - _window_start(t)) % STEP == x % STEP
    if kind == "hidden":                      # link[p] leads to q, which no parse visited (it lies inside a match)
        p, q = a
        return m.link[p] == p - q and not m.vis[q]
    if kind == "group":                       # positions of one warp step, one bucket, all keys different
        ps = a[0]
        t = ps[0] // TILE
        steps = {(p - _window_start(t)) // STEP for p in ps}
        keys = [d_key(b, p) for p in ps]
        return (len(steps) == 1 and all(p // TILE == t for p in ps) and len({d_mix(k)[0] for k in keys}) == 1
                and len(set(keys)) == len(keys))
    if kind == "nearest_bucket":              # q is the nearest earlier position of p's bucket, with another tag
        p, q = a
        bp = d_mix(d_key(b, p))
        between = [r for r in range(q + 1, p) if d_mix(d_key(b, r))[0] == bp[0]]
        bq = d_mix(d_key(b, q))
        return not between and bq[0] == bp[0] and bq[1] != bp[1]
    if kind == "chain_past_reach":            # p's bucket chain holds other tags within reach, its first equal tag past it
        p, r = a
        bp = d_mix(d_key(b, p))
        others = [q for q in range(p - REACH, p) if d_mix(d_key(b, q)) != bp and d_mix(d_key(b, q))[0] == bp[0]]
        equal = [q for q in range(max(0, p - REACH - 5000), p) if d_key(b, q) == d_key(b, p)]
        return len(others) >= 2 and equal and max(equal) == r and p - r > REACH
    if kind == "phase":                       # chunk c starts at bit phase v
        c, v = a
        return c < m.nch and m.cp[c][1] % 32 == v
    if kind == "chunk_at_match":
        c = a[0]
        syms = m.chunk_syms(c)
        return syms and syms[0][0] == c * CHUNK and syms[0][1] > 0
    if kind == "chunk_in_match":              # a match of `length` bytes runs across chunk c's first byte
        c, length = a
        return any(p < c * CHUNK < p + ln and ln == length for p, ln, _ in m.syms if ln)
    if kind == "chunk_in_literals":
        c = a[0]
        return all((m.sym(p) or (0, 1))[1] == 0 for p in (c * CHUNK - 1, c * CHUNK, c * CHUNK + 1))
    if kind == "eob_only":                    # the last chunk holds no symbol, only end-of-block
        return m.nch > 1 and not m.chunk_syms(m.nch - 1)
    if kind == "end_match":                   # the last match ends k bytes before the end
        k = a[0]
        last = [s for s in m.syms if s[1]]
        return bool(last) and last[-1][0] + last[-1][1] == m.n - k
    if kind == "bits_mod32":
        return m.bits % 32 == a[0]
    if kind == "out_len_mod4":
        return len(m.out) % 4 == a[0]
    if kind == "static":
        return not m.stored
    raise ValueError(kind)


# ---- Deflate catalogue -------------------------------------------------------------------------------------------------

def _halo_case(x, dist, seed):
    """destinations at t0 + x of tiles 1 and 2, sources `dist` back: at the halo's lane x when dist is REACH"""
    rng = random.Random(seed)
    L = Layout(2 * TILE + 400, seed)
    edges = []
    for t in (1, 2):
        key = high(rng, 3)
        p = t * TILE + x
        L.put(p - dist, key)
        L.dest(p, key)
        if dist == REACH:
            edges += [("tile", p, t, x), ("halo", p - dist, t, x), ("match", p, dist)]
        else:
            edges += [("tile", p, t, x), ("literal", p)]
    return L.data(), edges


def _hidden_case(seed, spots):
    """`spots`: (first, second, final) positions.  first = J K X (literals), second = J K X (a match over K, which is
    never visited), final = K: link[final] leads to the hidden K, the walk to the first K when it is within reach"""
    rng = random.Random(seed)
    L = Layout(2 * TILE + 2000, seed)
    edges = []
    for first, second, final in spots:
        j, k, x = high(rng, 3), high(rng, 3), high(rng, 3)
        L.put(first, j + k + x)
        L.dest(second, j + k + x)
        L.dest(final, k)
        hidden, src = second + 3, first + 3
        edges += [("match", second, second - first), ("hidden", final, hidden)]
        edges.append(("match", final, final - src) if final - src <= REACH else ("literal", final))
    return L.data(), edges


def _group_case(seed, ms, tile):
    """for each m of `ms`: m different keys of one bucket back to back inside one warp step, each with its source
    behind the step (sources in reverse order, so every chain passes the others)"""
    rng = random.Random(seed)
    t0 = tile * TILE
    at = t0 + 64 if tile else 8000          # the first group of a later tile finds its sources in the halo
    L = Layout(at + 8000 * len(ms) + 2000, seed)
    buckets = rng.sample(range(4096), len(ms))
    edges = []
    for m, bk in zip(ms, buckets):
        keys = d_bucket_keys(rng, bk, m)
        lane = 0 if m % 2 else 31 - 3 * (m - 1)
        base = at - (at - _window_start(tile)) % STEP + lane
        for j, k in enumerate(keys):
            L.put(base - 1500 - 700 * (m - j) - 37 * j, k)
        L.dest(base, b"".join(keys))
        ps = [base + 3 * j for j in range(m)]
        edges.append(("group", ps))
        for j, p in enumerate(ps):
            edges.append(("match", p, p - (base - 1500 - 700 * (m - j) - 37 * j)))
        at += 8000
    return L.data(), edges


def _bucket_reach_case(seed):
    """the nearest entry of p's bucket exactly REACH back with another tag, p's key further back: a literal; and a chain
    of other tags within reach whose first equal tag lies one past it"""
    rng = random.Random(seed)
    L = Layout(TILE + 4000, seed)
    p = TILE + 7
    # a bucket no filler key between the two uses
    busy = {d_mix(d_key(L.b, q))[0] for q in range(p - REACH - 8, p + 8)}
    a, bq = d_bucket_keys(rng, rng.choice(sorted(set(range(4096)) - busy)), 2)
    L.put(p - REACH - 3000, a)
    L.put(p - REACH, bq)
    L.dest(p, a)
    keys = d_bucket_keys(rng, rng.randrange(4096), 4)
    a2 = keys[0]
    p2 = TILE + 1500
    L.put(p2 - REACH - 1, a2)
    for j, k in enumerate(keys[1:]):
        L.put(p2 - 9000 * (j + 1) - 13, k)
    L.dest(p2, a2)
    return L.data(), [("nearest_bucket", p, p - REACH), ("literal", p), ("chain_past_reach", p2, p2 - REACH - 1),
                      ("literal", p2)]


def _phase_case(v, seed):
    """CHUNK literals, k of them 9-bit, so that chunk 1 starts at bit 3 + 8 CHUNK + k = v (mod 32); filler behind"""
    rng = random.Random(seed)
    k = (v - 3) % 32
    head = distinct_run(rng, CHUNK, high_at=rng.sample(range(CHUNK), k))
    return head + H.textlike(3000 + 37 * v, seed), [("phase", 1, v), ("literal", CHUNK - 1), ("static",)]


def _boundary_case(seed):
    """chunk 1 starts exactly at a match, chunk 2 inside a 258-byte match, chunk 3 inside a literal run"""
    rng = random.Random(seed)
    L = Layout(4 * CHUNK + 900, seed)
    key = high(rng, 3)
    L.put(700, key)
    L.dest(CHUNK, key)
    pat = high(rng, 260)
    L.put(1200, pat)
    L.dest(2 * CHUNK - 100, pat[:258] + GUARDS[-1:])
    L.put(3 * CHUNK - 10, distinct_run(rng, 20, high_at=range(20)))
    return L.data(), [("match", CHUNK, CHUNK - 700), ("chunk_at_match", 1), ("chunk_in_match", 2, 258),
                      ("chunk_in_literals", 3)]


def _tail_case(k, n, seed):
    """the last match ends k bytes before the end of n bytes; k = 0 with a match across the last chunk's start leaves
    that chunk only end-of-block"""
    rng = random.Random(seed)
    L = Layout(n, seed)
    pat = high(rng, 150)
    L.put(900, pat)
    start = n - 150 - k
    L.dest(start, pat[:150] + GUARDS[-1 - k:-1])
    edges = [("match", start, start - 900), ("end_match", k)]
    if k == 0 and start < (n - 1) // CHUNK * CHUNK:
        edges.append(("eob_only",))
    return L.data(), edges


def _bits_case(target, seed):
    """filler, then literals (8- and 9-bit) until the stream's bit count (kind "bits_mod32") or out_len (kind
    "out_len_mod4") reaches `target`"""
    kind, r = target
    rng = random.Random(seed)
    base = H.textlike(2 * CHUNK + 300 + 29 * seed % 500, seed)
    m = DeflateModel(base)
    for t in range(0, 8):
        for j in range(0, 32):
            bits = m.bits + 8 * t + 9 * j
            if (bits % 32 if kind == "bits_mod32" else (bits + 7) // 8 % 4) == r:
                order = rng.sample(range(t + j), j)
                return base + distinct_run(rng, t + j, high_at=order), [(kind, r)]
    raise AssertionError(target)


@functools.lru_cache(maxsize=None)
def deflate_cases():
    """(name, data, edges)"""
    out = []
    for x in (0, 1, 31, 32, 33):
        for dist in (REACH, REACH + 1):
            out.append((f"halo_x{x}_d{dist}", *_halo_case(x, dist, 100 + x + dist % 2)))
    out.append(("hidden_across_tiles", *_hidden_case(201, [(TILE - 20000, TILE - 100, TILE + 5),
                                                             (2 * TILE - 100, 2 * TILE + 50, 2 * TILE + 300)])))
    out.append(("hidden_reach_across_tiles", *_hidden_case(202, [(TILE - 32000, TILE - 50, TILE + 800),
                                                                   (2 * TILE - REACH + 2, 2 * TILE - 10, 2 * TILE + 5)])))
    out.append(("bucket_groups_2_5", *_group_case(301, (2, 3, 4, 5), 0)))
    out.append(("bucket_groups_6_8", *_group_case(302, (6, 7, 8), 0)))
    out.append(("bucket_groups_halo", *_group_case(303, (2, 5, 8), 1)))
    out.append(("bucket_reach", *_bucket_reach_case(304)))
    for v in range(32):
        out.append((f"phase_{v}", *_phase_case(v, 400 + v)))
    out.append(("chunk_boundaries", *_boundary_case(500)))
    out.append(("tail_eob_only", *_tail_case(0, 4 * CHUNK + 40, 501)))
    out.append(("tail_end_n", *_tail_case(0, 3 * CHUNK + 1000, 502)))
    out.append(("tail_end_n_1", *_tail_case(1, 3 * CHUNK + 1001, 503)))
    out.append(("tail_end_n_2", *_tail_case(2, 3 * CHUNK + 2, 504)))
    for k, tgt in enumerate([("bits_mod32", 0), ("out_len_mod4", 0), ("out_len_mod4", 1), ("out_len_mod4", 2),
                             ("out_len_mod4", 3)]):
        out.append((f"{tgt[0]}_{tgt[1]}", *_bits_case(tgt, 600 + k)))
    return tuple(out)


DEFLATE_VARIANTS = ("halo_short", "bucket", "late_checkpoint")


# ---- LZ4 model ---------------------------------------------------------------------------------------------------------

class LZ4Model:
    """lz4c_chain_kernel's links and lz4c_parse_kernel's parse over the window dictionary + block"""

    def __init__(self, block, dictionary=b"", variant=None):
        d = bytes(dictionary)[-MAX_DICT:] if len(dictionary) > MAX_DICT else bytes(dictionary)
        self.d = dl = len(d)
        b = self.b = d + bytes(block)
        w = self.w = len(b)
        nk = w - 3 if w >= 4 else 0
        keys = self.keys = [l_key(b, p) for p in range(nk)]
        link, last = [0] * nk, {}
        for p in range(nk):
            h = l_bucket(keys[p])
            q = last.get(h)
            if q is not None and p - q <= L_REACH:
                link[p] = p - q
            last[h] = p
        self.bucket_link = list(link)
        bases = range(0, nk, STEP) if variant == "front_to_back" else range((nk - 1) // STEP * STEP, -1, -STEP)
        for base in bases:
            new = {}
            for p in range(base, min(base + STEP, nk)):
                dd = link[p]
                if dd and variant != "bucket":
                    q = p - dd
                    while True:
                        if keys[q] == keys[p]:
                            dd = p - q
                            break
                        nx = link[q]
                        if nx == 0 or p - (q - nx) > L_REACH:
                            dd = 0
                            break
                        q -= nx
                if variant == "write_first":
                    link[p] = dd
                else:
                    new[p] = dd
            for p, dd in new.items():
                link[p] = dd
        self.link = link
        vis = self.vis = bytearray(w + 1)
        for p in range(dl - 4 if dl >= 4 else 0):
            vis[p] = 1
        seqs, i, lit0 = [], dl, dl
        while i < w - 9:
            q, dd, found = i, link[i], False
            while dd:
                q -= dd
                if i - q > L_REACH:
                    break
                if vis[q]:
                    found = True
                    break
                dd = link[q]
            vis[i] = 1
            if not found:
                i += 1
                continue
            ln = 4
            while i + ln < w - 5 and b[i + ln] == b[q + ln]:
                ln += 1
            if w - i < 12:
                break
            seqs.append((i, ln, i - q, b[lit0:i]))
            i += ln
            lit0 = i
        self.seqs = seqs
        self.at = {s[0]: s for s in seqs}
        self.out = H.lz4_block_from_sequences([(s[3], s[1], s[2]) for s in seqs], b[lit0:], b[:dl])[0]


def lz4_model(block, dictionary=b"", variant=None):
    return LZ4Model(block, dictionary, variant).out


def lz4_edge(m, e):
    """True when the model reaches edge `e` (positions are window positions: the dictionary comes first)"""
    kind, a = e[0], e[1:]
    if kind == "match":
        s = m.at.get(a[0])
        return s is not None and s[2] == a[1]
    if kind == "literal":
        return m.d <= a[0] < m.w and a[0] not in m.at and m.vis[a[0]] and not any(
            s[0] < a[0] < s[0] + s[1] for s in m.seqs)
    if kind == "between":                     # p -> q -> r down p's bucket chain, q another key with no earlier copy
        p, q, r = a
        k = m.keys
        return (m.bucket_link[p] == p - q and m.bucket_link[q] == q - r and k[p] == k[r] != k[q]
                and k[q] not in k[max(0, q - L_REACH):q])
    if kind == "steps":                       # p at lane lp, q at lane lq, `apart` warp steps before p's
        p, lp, q, lq, apart = a
        return p % STEP == lp and q % STEP == lq and p // STEP - q // STEP == apart
    if kind == "chain_other_keys":            # p's bucket chain passes n other keys before its key at distance dist
        p, n, dist = a
        others, q = 0, p
        while m.bucket_link[q]:
            q -= m.bucket_link[q]
            if m.keys[q] == m.keys[p]:
                return others >= n and p - q == dist
            others += 1
        return False
    if kind == "group":
        ps = a[0]
        keys = [m.keys[p] for p in ps]
        return (len({p // STEP for p in ps}) == 1 and len({l_bucket(k) for k in keys}) == 1
                and len(set(keys)) == len(keys))
    if kind == "seam":                        # p's key straddles the dictionary / block seam, and no parse visits it
        p = a[0]
        return m.d - 3 <= p < m.d and not m.vis[p]
    if kind == "link":
        p, q = a
        return m.link[p] == p - q
    if kind == "align":
        return m.d % STEP == a[0]
    raise ValueError(kind)


# ---- LZ4 catalogue -----------------------------------------------------------------------------------------------------

def _between_case(seed, spots):
    """for each (lane of p, lane of q, steps apart): r (key A) -> q (key B, same bucket, no earlier B) -> p (key A);
    r is reachable from p only through q's bucket link"""
    rng = random.Random(seed)
    L = Layout(3000, seed)
    used, edges = set(), []
    at = 200
    for lp, lq, apart in spots:
        bk, (ka, kb) = l_bucket_keys(rng, 2, used)
        used.add(bk)
        q = (at // STEP) * STEP + lq
        p = (q // STEP + apart) * STEP + lp
        assert p >= q + 5
        r = q - 23
        L.put(r, ka)
        L.put(q, kb)
        L.dest(p, ka)
        edges += [("between", p, q, r), ("steps", p, lp, q, lq, apart), ("match", p, p - r)]
        at = p + 3 * STEP
    return L.data(), edges


def _reach_case(seed, dist):
    """p's key `dist` back behind three other keys of its bucket on the chain"""
    rng = random.Random(seed)
    p = dist + 400
    L = Layout(p + 300, seed)
    _, keys = l_bucket_keys(rng, 4)
    L.put(p - dist, keys[0])
    for j, k in enumerate(keys[1:]):
        L.put(p - dist + 20000 * (j + 1) + 11 * j, k)
    L.dest(p, keys[0])
    return L.data(), [("chain_other_keys", p, 3, dist), ("match", p, dist) if dist <= L_REACH else ("literal", p)]


def _lz4_group_case(seed, ms):
    rng = random.Random(seed)
    L = Layout(5000 * (len(ms) + 1) + 2000, seed)
    used, edges = set(), []
    at = 5000
    for m in ms:
        bk, keys = l_bucket_keys(rng, m, used)
        used.add(bk)
        base = (at // STEP) * STEP + (0 if m == 8 else (STEP - 4 * m) if m % 2 else 1)
        srcs = [base - 900 - 400 * (m - j) - 29 * j for j in range(m)]
        for s, k in zip(srcs, keys):
            L.put(s, k)
        L.dest(base, b"".join(keys))
        ps = [base + 4 * j for j in range(m)]
        edges.append(("group", ps))
        edges += [("match", p, p - s) for p, s in zip(ps, srcs)]
        at += 5000
    return L.data(), edges


def _seam_case(seed, dlen, blen=400):
    """a dictionary of dlen bytes whose window ends inside key A (A straddles the seam, so it is never visited), A once
    more well inside the dictionary, and A in the block: the walk passes the straddling copy to the visited one; and
    a key near the block's start whose source lies in the dictionary"""
    rng = random.Random(seed)
    wd = min(dlen, MAX_DICT)
    L = Layout(wd + blen, seed)
    a, c = high(rng, 4), high(rng, 4)
    split = 1 + seed % 3                   # A's bytes in the dictionary
    s = wd - split
    src = wd - 200 - seed % 40
    L.put(src, a)
    L.put(s, a)
    L.put(wd - 120, c)
    L.dest(wd + 8, c)
    L.dest(wd + 150, a)
    win = L.data()
    head = H.textlike(dlen - wd, seed + 1) if dlen > wd else b""
    edges = [("seam", s), ("link", wd + 150, s), ("match", wd + 150, wd + 150 - src), ("match", wd + 8, 128),
             ("align", wd % STEP)]
    return win[wd:], head + win[:wd], edges


@functools.lru_cache(maxsize=None)
def lz4_cases():
    """(name, block, dictionary, edges)"""
    out = []
    for k, (name, spots) in enumerate((("between_in_step", [(31, 0, 0), (12, 5, 0), (31, 26, 0)]),
                                       ("between_across_steps", [(0, 26, 1), (3, 20, 1), (31, 0, 1), (0, 31, 2)]))):
        data, edges = _between_case(700 + k, spots)
        out.append((name, data, b"", edges))
    for dist in (L_REACH, L_REACH + 1):
        data, edges = _reach_case(710 + dist % 2, dist)
        out.append((f"reach_chain_{dist}", data, b"", edges))
    data, edges = _lz4_group_case(720, (2, 3, 4, 5, 6, 7, 8))
    out.append(("bucket_groups", data, b"", edges))
    for s in range(1, 32):
        block, d, edges = _seam_case(800 + s, 256 + s)
        out.append((f"seam_align_{s}", block, d, edges))
    for dlen in (MAX_DICT - 1, MAX_DICT, MAX_DICT + 1):
        block, d, edges = _seam_case(900 + dlen % 7, dlen)
        out.append((f"seam_dict_{dlen}", block, d, edges))
    return tuple(out)


LZ4_VARIANTS = ("write_first", "front_to_back", "bucket")
