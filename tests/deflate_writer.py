"""A test-only Deflate writer (RFC 1951) that writes chosen streams: block types, code sets, header encodings, symbol
spellings and symbols a valid stream never contains.

Codes are assigned the way the oracle's swco_tree_build does (oracle/huffman.c): symbols sorted by (length, symbol), a
counter that starts at -1, is incremented per symbol and shifted left when the length grows; the low `length` bits of the
counter are the code, sent most significant bit first.  For a set whose Kraft sum is over 1 the counter runs past the
code space and wraps, and the decoder keeps the shortest prefix (among equal paths, the code assigned last): `Code`
emulates that, and the writer refuses to send a symbol that such a decoder would not read back.

The writer records a `Trace` of what it sent, so that tests can assert what a stream covers without decoding it."""
from fractions import Fraction

LEN_BASE = [3, 4, 5, 6, 7, 8, 9, 10, 11, 13, 15, 17, 19, 23, 27, 31, 35, 43, 51, 59, 67, 83, 99, 115, 131, 163, 195, 227, 258]
LEN_EXTRA = [0] * 8 + [1] * 4 + [2] * 4 + [3] * 4 + [4] * 4 + [5] * 4 + [0]
DIST_BASE = [1, 2, 3, 4, 5, 7, 9, 13, 17, 25, 33, 49, 65, 97, 129, 193, 257, 385, 513, 769, 1025, 1537, 2049, 3073, 4097,
             6145, 8193, 12289, 16385, 24577]
DIST_EXTRA = [0, 0, 0, 0] + [k // 2 for k in range(2, 28)]
CL_ORDER = [16, 17, 18, 0, 8, 7, 9, 6, 10, 5, 11, 4, 12, 3, 13, 2, 14, 1, 15]
FIXED_LIT = [8] * 144 + [9] * 112 + [7] * 24 + [8] * 8
FIXED_DIST = [5] * 32


def len_symbol(length):
    """(symbol, extra value) of a match length, the RFC spelling (258 is 285)"""
    if length == 258:
        return 285, 0
    s = max(i for i in range(28) if LEN_BASE[i] <= length)
    return 257 + s, length - LEN_BASE[s]


def dist_symbol(dist):
    s = max(i for i in range(30) if DIST_BASE[i] <= dist)
    return s, dist - DIST_BASE[s]


class Code:
    """Canonical code of a list of code lengths (index = symbol), as the oracle assigns it."""

    def __init__(self, lengths):
        self.lengths = list(lengths)
        self.codes = {}                       # symbol -> code (the low `length` bits of the counter)
        slots = {}                            # (length, code) -> symbol assigned last to that path
        counter, loop = -1, -1
        for L in range(1, max(self.lengths, default=0) + 1):
            for s, ls in enumerate(self.lengths):
                if ls != L:
                    continue
                counter += 1
                if L != loop:
                    counter <<= L - loop
                    loop = L
                self.codes[s] = counter & ((1 << L) - 1)
                slots[(L, self.codes[s])] = s
        self.slots = slots
        self.kraft = sum((Fraction(1, 1 << L) for L in self.lengths if L), Fraction(0))

    def reads_back(self, s):
        """True when the oracle's decoder reads symbol s's code back as s"""
        L = self.lengths[s] if s < len(self.lengths) else 0
        if not L:
            return False
        c = self.codes[s]
        return self.slots[(L, c)] == s and not any((k, c >> (L - k)) in self.slots for k in range(1, L))


# ------------------------------------------------------------------------------------------------------ length sets
def as_list(lens, size):
    """{symbol: length} -> list of `size` lengths"""
    out = [0] * size
    for s, L in lens.items():
        out[s] = L
    return out


def staircase(symbols):
    """lengths 1, 2, ..., n-1, n-1 for n <= 16 symbols in the given order: a complete set whose longest codes are n-1 bits;
    the last symbol in symbol order among the two longest gets the all-ones code"""
    n = len(symbols)
    assert 2 <= n <= 16
    return {s: min(i + 1, n - 1) for i, s in enumerate(symbols)}


def flat(symbols, short_first=True):
    """a complete set over n >= 2 symbols: 2^k - n codes of k-1 bits, the rest k bits (k = ceil(log2 n))"""
    symbols = list(symbols)
    n = len(symbols)
    assert n >= 2
    k = (n - 1).bit_length()
    nshort = (1 << k) - n
    order = symbols if short_first else symbols[::-1]
    return {s: (k - 1 if i < nshort else k) for i, s in enumerate(order)}


def huffman(freqs, maxlen):
    """code lengths of a complete Huffman code over the symbols with a non-zero count, limited to `maxlen` bits (when the
    plain Huffman code is longer a flat code is used)"""
    import heapq
    used = [s for s, f in freqs.items() if f]
    if len(used) < 2:
        return flat(used + [x for x in range(2) if x not in used][:2 - len(used)])
    heap = [(f, i, [s]) for i, (s, f) in enumerate((s, freqs[s]) for s in used)]
    heapq.heapify(heap)
    depth = {s: 0 for s in used}
    k = len(heap)
    while len(heap) > 1:
        f1, _, a = heapq.heappop(heap)
        f2, _, b = heapq.heappop(heap)
        for s in a + b:
            depth[s] += 1
        heapq.heappush(heap, (f1 + f2, k, a + b))
        k += 1
    if max(depth.values()) > maxlen:
        return flat(used)
    return depth


def kraft(lens):
    return sum((Fraction(1, 1 << L) for L in (lens.values() if isinstance(lens, dict) else lens) if L), Fraction(0))


def oversubscribe(lens, limit, maxlen=15):
    """the complete set `lens` ({symbol: length}) plus one unused code that pushes the Kraft sum over 1 without changing
    what any used code decodes to: it is assigned last (one bit longer than the longest code, or as long as the longest with a
    symbol above all of them when `maxlen` forbids longer), so its wrapped code sits behind a shorter prefix.  `limit`:
    symbols must be below it."""
    assert kraft(lens) == 1, "only a complete set can be over-subscribed by one code"
    top = max(lens.values())
    free = [s for s in range(limit) if s not in lens]
    if top < maxlen:
        extra, L = free[-1], top + 1
    else:
        above = [s for s in free if s > max(s2 for s2, L2 in lens.items() if L2 == top)]
        assert above, "no unused symbol sorts after the longest codes"
        extra, L = above[-1], top
    out = dict(lens)
    out[extra] = L
    assert kraft(out) > 1
    return out


# ------------------------------------------------------------------------------------------------------ tokens
class Match:
    """A match of `length` bytes at distance `dist`.  lsym / lextra and dsym / dextra pick the spelling (258 as 284 + 31);
    `unchecked` lets the distance reach before the output's start."""
    __slots__ = ("length", "dist", "lsym", "lextra", "dsym", "dextra", "unchecked")

    def __init__(self, length, dist, lsym=None, lextra=None, dsym=None, dextra=None, unchecked=False):
        if lsym is None:
            lsym, lextra = len_symbol(length)
        if dsym is None and dist is not None:
            dsym, dextra = dist_symbol(dist)
        self.length, self.dist, self.lsym, self.lextra, self.dsym, self.dextra = length, dist, lsym, lextra, dsym, dextra
        self.unchecked = unchecked


class Raw:
    """A lit/len symbol (and, for a length symbol, a distance symbol) written as is, with `extra` bits after each:
    286/287, distance codes 30/31.  The stream fails at it, so it carries no output."""
    __slots__ = ("lsym", "lextra", "dsym", "dextra")

    def __init__(self, lsym, lextra=0, dsym=None, dextra=0):
        self.lsym, self.lextra, self.dsym, self.dextra = lsym, lextra, dsym, dextra


class Trace:
    """What a writer emitted.  Bit offsets count from the first bit of the first byte (start bits included).
    - lengths: {(alphabet, code length)} of every symbol written ('lit', 'dist', 'cl'); all_ones: alphabets in which the
      all-ones 15-bit code was written
    - symbols: (alphabet, symbol, code length, bit offset) of every symbol except the literals of literal runs (bytes tokens)
    - matches: (length, dist, literal run before it, lsym, lextra, dsym, dextra, first bit, end bit)
    - extras: (alphabet, width, bit offset) of every extra-bit field of a match
    - blocks: (type, first bit, first bit of the symbols, end bit, oversubscribed alphabets)
    - codes: {first bit of a block's symbols: (lit/len Code, distance Code)}"""

    def __init__(self):
        self.start_bits = 0
        self.lengths, self.all_ones = set(), set()
        self.symbols, self.matches, self.blocks, self.extras = [], [], [], []
        self.codes = {}


class BitWriter:
    def __init__(self):
        self.out = bytearray()
        self.acc = 0
        self.n = 0
        self.pos = 0

    def bits(self, v, n):
        """n bits of v, least significant first"""
        self.acc |= (v & ((1 << n) - 1)) << self.n
        self.n += n
        self.pos += n
        if self.n >= 8:
            k = self.n >> 3
            self.out += (self.acc & ((1 << (8 * k)) - 1)).to_bytes(k, "little")
            self.acc >>= 8 * k
            self.n -= 8 * k

    def code(self, c, L):
        """a Huffman code, most significant bit first"""
        self.bits(int(format(c, f"0{L}b")[::-1], 2) if L else 0, L)

    def align(self):
        self.bits(0, (-self.pos) & 7)

    def data(self):
        return bytes(self.out) + (bytes([self.acc]) if self.n else b"")


class DeflateWriter:
    """Writes blocks one after another; `out` is the output a decoder should produce.

    oversub: None, 'lit', 'dist' or 'cl' — every dynamic block (and every fixed block, written as a dynamic block with
    complete code sets of the symbols it uses) gets that alphabet over-subscribed by one unused code (`oversubscribe`)."""

    def __init__(self, oversub=None, start_bits=0, junk=0):
        self.w = BitWriter()
        self.w.bits(junk, start_bits)     # the stream starts `start_bits` into its first byte; stored blocks align to bytes
        self.out = bytearray()
        self.run = 0                      # literal bytes since the last match
        self.trace = Trace()
        self.trace.start_bits = start_bits
        self.oversub = oversub

    # ---- blocks
    def stored(self, data, final=False, length=None, nlength=None):
        start = self.w.pos
        self.w.bits(int(final), 1)
        self.w.bits(0, 2)
        self.w.align()
        ln = len(data) if length is None else length
        self.w.bits(ln, 16)
        self.w.bits((~ln & 0xFFFF) if nlength is None else nlength, 16)
        self.w.bits(int.from_bytes(data, "little"), 8 * len(data))
        self.out += data
        self.run += len(data)
        self.trace.blocks.append(("stored", start, None, self.w.pos, ()))

    def fixed(self, tokens, final=False, eob=True):
        if self.oversub:
            return self.dynamic(tokens, final=final, eob=eob)
        start = self.w.pos
        self.w.bits(int(final), 1)
        self.w.bits(1, 2)
        self._symbols(tokens, Code(FIXED_LIT), Code(FIXED_DIST), eob, start, "fixed")

    def dynamic(self, tokens, lit_lens=None, dist_lens=None, final=False, eob=True, hlit=None, hdist=None, hclen=None,
                cl_lens=None, cl_ops=None, header_only=False):
        """lit_lens / dist_lens: lists indexed by symbol (None: complete sets built from the tokens' symbol counts).
        hlit / hdist / hclen: the header counts (defaults: as few as the lengths need); cl_ops: the code-length symbols,
        each a length 0..15 or (16 | 17 | 18, repeat count) (default: runs of zeros as 17/18, repeats as 16); cl_lens:
        the 19 code-length code lengths (default: a complete set over the symbols cl_ops uses)."""
        start = self.w.pos
        if lit_lens is None or dist_lens is None:
            freq_l, freq_d = self._used(tokens, eob)
            if lit_lens is None:
                lit_lens = as_list(huffman(freq_l, 15), 286)
            if dist_lens is None:
                dist_lens = as_list(huffman(freq_d, 15), 30)
        lit_lens, dist_lens = list(lit_lens), list(dist_lens)
        over = ()
        if self.oversub == "lit":
            lit_lens = as_list(oversubscribe({s: L for s, L in enumerate(lit_lens) if L}, 286), max(len(lit_lens), 286))
            over = ("lit",)
        elif self.oversub == "dist":
            dist_lens = as_list(oversubscribe({s: L for s, L in enumerate(dist_lens) if L}, 32), 32)
            over = ("dist",)
        if hlit is None:
            hlit = max(257, max((s + 1 for s, L in enumerate(lit_lens) if L), default=0))
        if hdist is None:
            hdist = max(1, max((s + 1 for s, L in enumerate(dist_lens) if L), default=0))
        lens = (lit_lens + [0] * 288)[:hlit] + (dist_lens + [0] * 32)[:hdist]
        if cl_ops is None:
            cl_ops = rle(lens)
        if cl_lens is None or cl_lens == "staircase":
            freq = {}
            for op in cl_ops:
                s = op if isinstance(op, int) else op[0]
                freq[s] = freq.get(s, 0) + 1
            cl = staircase(sorted(freq)) if cl_lens == "staircase" else flat(sorted(freq)) if len(freq) > 1 else {next(iter(freq)): 1, (1 if 0 in freq else 0): 1}
            if self.oversub == "cl":
                cl = oversubscribe(cl, 19, 7)
                over = ("cl",)
            cl_lens = as_list(cl, 19)
        if hclen is None:
            hclen = max(4, max((i + 1 for i, s in enumerate(CL_ORDER) if cl_lens[s]), default=0))
        w = self.w
        w.bits(int(final), 1)
        w.bits(2, 2)
        w.bits(hlit - 257, 5)
        w.bits(hdist - 1, 5)
        w.bits(hclen - 4, 4)
        for i in range(hclen):
            w.bits(cl_lens[CL_ORDER[i]], 3)
        clc = Code([cl_lens[s] if CL_ORDER.index(s) < hclen else 0 for s in range(19)])
        for op in cl_ops:
            s, reps = (op, None) if isinstance(op, int) else op
            self._put(clc, s, "cl")
            if s == 16:
                w.bits(reps - 3, 2)
            elif s == 17:
                w.bits(reps - 3, 3)
            elif s == 18:
                w.bits(reps - 11, 7)
        if header_only:
            self.trace.blocks.append(("dynamic", start, None, w.pos, over))
            return
        self._symbols(tokens, Code(lit_lens[:hlit]), Code(dist_lens[:hdist]), eob, start, "dynamic", over)

    def bits(self, v, n):
        """raw bits (a stream that ends inside a field)"""
        self.w.bits(v, n)

    def finish(self):
        """-> (bytes, bit position after the stream's last bit, counting the start bits)"""
        return self.w.data(), self.w.pos

    # ---- symbols
    @staticmethod
    def _used(tokens, eob):
        lit, dist = {}, {}
        def add(d, s):
            d[s] = d.get(s, 0) + 1
        for t in tokens:
            if isinstance(t, int):
                add(lit, t)
            elif isinstance(t, (bytes, bytearray)):
                for b in set(t):
                    add(lit, b)
            else:
                add(lit, t.lsym)
                if t.dsym is not None:
                    add(dist, t.dsym)
        if eob:
            add(lit, 256)
        return lit, dist

    def _put(self, code, s, alphabet, raw=False):
        if not raw and not code.reads_back(s):
            raise ValueError(f"{alphabet} symbol {s} has no code the decoder reads back")
        L = code.lengths[s] if s < len(code.lengths) else 0
        if not L:
            raise ValueError(f"{alphabet} symbol {s} has no code")
        pos = self.w.pos
        self.w.code(code.codes[s], L)
        self.trace.lengths.add((alphabet, L))
        if L == 15 and code.codes[s] == (1 << 15) - 1:
            self.trace.all_ones.add(alphabet)
        self.trace.symbols.append((alphabet, s, L, pos))

    def _symbols(self, tokens, lit, dist, eob, start, kind, over=()):
        sym0 = self.w.pos
        self.trace.codes[sym0] = (lit, dist)
        w, out = self.w, self.out
        for t in tokens:
            if isinstance(t, int):
                self._put(lit, t, "lit")
                out.append(t)
                self.run += 1
            elif isinstance(t, (bytes, bytearray)):
                code = [""] * 256                     # each literal's code in the order the bits are written
                for b in set(t):
                    if not lit.reads_back(b):
                        raise ValueError(f"literal {b} has no code the decoder reads back")
                    L = lit.lengths[b]
                    code[b] = format(lit.codes[b], f"0{L}b")
                    self.trace.lengths.add(("lit", L))
                    if L == 15 and lit.codes[b] == (1 << 15) - 1:
                        self.trace.all_ones.add("lit")
                if t:
                    bits = "".join(code[b] for b in t)
                    w.bits(int(bits[::-1], 2), len(bits))
                out += t
                self.run += len(t)
            elif isinstance(t, Raw):
                self._put(lit, t.lsym, "lit", raw=True)
                if 257 <= t.lsym <= 285:
                    w.bits(t.lextra, LEN_EXTRA[t.lsym - 257])
                if t.dsym is not None:
                    self._put(dist, t.dsym, "dist", raw=True)
                    w.bits(t.dextra, DIST_EXTRA[t.dsym] if t.dsym < 30 else 0)
            else:
                assert LEN_BASE[t.lsym - 257] + t.lextra == t.length and t.lextra < (1 << LEN_EXTRA[t.lsym - 257])
                assert DIST_BASE[t.dsym] + t.dextra == t.dist and t.dextra < (1 << DIST_EXTRA[t.dsym])
                if not t.unchecked:
                    assert t.dist <= len(out), "distance beyond the output so far"
                p0 = w.pos
                self._put(lit, t.lsym, "lit")
                self.trace.extras.append(("lit", LEN_EXTRA[t.lsym - 257], w.pos))
                w.bits(t.lextra, LEN_EXTRA[t.lsym - 257])
                self._put(dist, t.dsym, "dist")
                self.trace.extras.append(("dist", DIST_EXTRA[t.dsym], w.pos))
                w.bits(t.dextra, DIST_EXTRA[t.dsym])
                self.trace.matches.append((t.length, t.dist, self.run, t.lsym, t.lextra, t.dsym, t.dextra, p0, w.pos))
                if t.dist <= len(out):
                    if t.dist >= t.length:
                        out += out[len(out) - t.dist:len(out) - t.dist + t.length]
                    else:
                        for _ in range(t.length):
                            out.append(out[-t.dist])
                self.run = 0
        if eob:
            self._put(lit, 256, "lit")
        self.trace.blocks.append((kind, start, sym0, w.pos, over))


def rle(lens):
    """code-length symbols for a list of lengths: zero runs as 17 / 18, repeats of the previous length as 16"""
    ops, i, n = [], 0, len(lens)
    while i < n:
        v = lens[i]
        j = i
        while j < n and lens[j] == v:
            j += 1
        k = j - i
        if v == 0:
            while k >= 11:
                r = min(k, 138)
                ops.append((18, r))
                k -= r
            if k >= 3:
                ops.append((17, k))
                k = 0
            ops += [0] * k
        else:
            ops.append(v)
            k -= 1
            while k >= 3:
                r = min(k, 6)
                ops.append((16, r))
                k -= r
            ops += [v] * k
        i = j
    return ops


# inflate_warp.cu: WIN_WORDS = 19 32-bit words per lane window, 32 windows (one per lane) per chunk.  test_deflate_writer.py
# reads WIN_WORDS from the kernel source and fails when the two part.
K1W_WIN_WORDS = 19
K1W_WIN_BITS = 32 * K1W_WIN_WORDS


def k1w_window_offsets(trace, block, win_bits=K1W_WIN_BITS, windows=32):
    """Where the warp decoder's windows put each match of a block.  The decoder stages the symbol stream in chunks of
    `windows` windows of `win_bits` bits; a chunk starts where the previous one's last token ended, that token being the
    first to end at or beyond the chunk's limit.  Needs every token of the block in the trace (no literal runs written as
    bytes tokens).  -> [(offset of the match inside its window, chunk index, the match crosses the chunk's limit)]"""
    _, _, sym0, end, _ = block
    toks = {(m[7], m[8]) for m in trace.matches if sym0 <= m[7] < end}
    inside = sorted(toks)
    events = sorted(toks | {(s[3], s[3] + s[2]) for s in trace.symbols
                            if s[0] == "lit" and sym0 <= s[3] < end and not _covered(inside, s[3])})
    out, base, chunk = [], sym0, 0
    for a, b in events:
        limit = base + win_bits * windows
        assert a < limit, "a token is missing from the trace"
        if (a, b) in toks:
            out.append(((a - base) % win_bits, chunk, b >= limit))
        if b >= limit:
            base, chunk = b, chunk + 1
    return out


def _covered(spans, p):
    import bisect
    i = bisect.bisect_right(spans, (p, float("inf"))) - 1
    return i >= 0 and spans[i][0] <= p < spans[i][1]
