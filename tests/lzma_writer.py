"""Test-only LZMA / LZMA2 writer and a model of the reference's decoder.

The writer encodes decoder-level operations -- literal bytes, matches (length, rep0), rep0..rep3 with a length, short reps
and the end marker -- through the same adaptive model the decoder uses, so it can write what no encoder writes: lc + lp up
to 12 (and raw lc / lp / pb past what a properties byte can hold), distances past the dictionary, lengths past the known size,
symbols behind the end marker, a flush that leaves the range decoder's code non-zero, a first byte other than 0.  The LZMA2
layer writes chunks with any control byte, reset kind, properties byte, declared sizes and stored payload.

The expected answer is not taken from the oracle: `decode_lzma` / `decode_lzma2` restate Sources/LZMA/LZMADecoder.swift,
LZMARangeDecoder.swift, LZMALenDecoder.swift, LZMABitTreeDecoder.swift and Sources/LZMA2/LZMA2Decoder.swift, including
what they do on input no encoder writes: `dictStart` / `dictEnd`, `byte(at:)` with its wrapped branch, the flat 432-entry
`probabilities` array that isRep0Long at state 11 / posState 15 indexes one past its end, 16 length coders per length
decoder, and Swift's `>>` (a negative count shifts left).  Array bounds and reads past the input are traps.  Each decoded
symbol is recorded in a trace for the coverage assertions."""

OK, OVERFLOW, TRAP, UNSUPPORTED = 0, 1, 2, 6
WRONG_PROPERTIES, INIT_ERROR, EXCEEDED, WINDOW_EMPTY, FINISH_ERROR, REPEAT_EXCEED, NOT_ENOUGH = 301, 302, 303, 304, 305, 306, 307
WRONG_DICT, WRONG_CONTROL, WRONG_RESET, WRONG_SIZES = 401, 402, 403, 404

TOP = 1 << 24
END_MARKER = 0xFFFFFFFF


class Fail(Exception):
    """the reference throws `code`; TRAP stands for a precondition or array-bounds trap"""

    def __init__(self, code):
        super().__init__(code)
        self.code = code


def swift_shr(x, n):
    """Swift's smart shift `x >> n` on Int: a negative count shifts left"""
    return x >> n if n >= 0 else x << -n


def pos_slot_of(rep0):
    if rep0 < 4:
        return rep0
    n = rep0.bit_length()
    return 2 * (n - 1) + ((rep0 >> (n - 2)) & 1)


# ------------------------------------------------------------------------------------------------------------ coders
class RangeEncoder:
    def __init__(self):
        self.low, self.range, self.cache, self.cache_size = 0, 0xFFFFFFFF, 0, 1
        self.out = bytearray()

    def _shift_low(self):
        if self.low < 0xFF000000 or self.low >= 1 << 32:
            carry = self.low >> 32
            temp = self.cache
            while True:
                self.out.append((temp + carry) & 0xFF)
                temp = 0xFF
                self.cache_size -= 1
                if self.cache_size == 0:
                    break
            self.cache = (self.low >> 24) & 0xFF
        self.cache_size += 1
        self.low = (self.low & 0x00FFFFFF) << 8

    def _norm(self):
        while self.range < TOP:
            self.range = (self.range << 8) & 0xFFFFFFFF
            self._shift_low()

    def bit(self, arr, i, want):
        p = arr[i]
        bound = (self.range >> 11) * p
        if want == 0:
            self.range = bound
            arr[i] = p + ((2048 - p) >> 5)
        else:
            self.low += bound
            self.range -= bound
            arr[i] = p - (p >> 5)
        self._norm()
        return want

    def direct(self, count, want):
        for i in range(count - 1, -1, -1):
            self.range >>= 1
            if (want >> i) & 1:
                self.low += self.range
            self._norm()
        return want

    def finish(self, extra=0):
        """flush; `extra` (< the final range) moves the coded value up, which leaves the decoder's code == extra"""
        assert 0 <= extra < self.range
        self.low += extra
        for _ in range(5):
            self._shift_low()
        return bytes(self.out)


class Reader:
    """LittleEndianByteReader over data[start:]; reading past the end traps"""

    def __init__(self, data, pos=0):
        self.data, self.pos = data, pos

    def left(self):
        return len(self.data) - self.pos

    def byte(self):
        if self.pos >= len(self.data):
            raise Fail(TRAP)
        b = self.data[self.pos]
        self.pos += 1
        return b


class RangeDecoder:
    """LZMARangeDecoder.swift:20-80"""

    def __init__(self, rd):
        if rd.left() < 5:
            raise Fail(INIT_ERROR)
        self.rd = rd
        b = rd.byte()
        self.code = int.from_bytes(bytes(rd.byte() for _ in range(4)), "big")
        self.range = 0xFFFFFFFF
        if b != 0:
            raise Fail(INIT_ERROR)

    def _norm(self):
        if self.range < TOP:
            self.range = (self.range << 8) & 0xFFFFFFFF
            self.code = ((self.code << 8) & 0xFFFFFFFF) | self.rd.byte()

    def bit(self, arr, i, want=None):
        p = arr[i]
        bound = (self.range >> 11) * p
        if self.code < bound:
            arr[i] = p + ((2048 - p) >> 5)
            self.range = bound
            b = 0
        else:
            arr[i] = p - (p >> 5)
            self.code -= bound
            self.range -= bound
            b = 1
        self._norm()
        return b

    def direct(self, count, want=None):
        res = 0
        while True:                          # repeat-while: at least one pass
            self.range >>= 1
            self.code = (self.code - self.range) & 0xFFFFFFFF
            t = (0 - (self.code >> 31)) & 0xFFFFFFFF
            self.code = (self.code + (self.range & t)) & 0xFFFFFFFF
            self._norm()
            res = ((res << 1) + t + 1) & 0xFFFFFFFF
            count -= 1
            if count <= 0:
                break
        return res


# ------------------------------------------------------------------------------------------------------------ model
class Model:
    """LZMADecoder's state.  The writer keeps one to choose each bit's probability; the decoder model keeps another."""

    def __init__(self, lc=3, lp=0, pb=2, dict_size=1 << 24):
        self.lc, self.lp, self.pb, self.dict_size = lc, lp, pb, dict_size
        self.out = bytearray()
        self.dict_start = self.dict_end = 0
        self.ready = False
        self.state = 0
        self.reps = [0, 0, 0, 0]
        self.trace = []
        self.chunk = None                    # input offset of the LZMA2 chunk being decoded
        self.controls = []                   # input offset of every LZMA2 control byte
        self.wide = None                     # output length when a decode() with lc + lp > 4 first got past its range coder

    def reset(self):
        """resetStateAndDecoders() LZMADecoder.swift:79-100"""
        self.state = 0
        self.reps = [0, 0, 0, 0]
        self.probs = [1024] * 432
        n = swift_shl(1, self.lc + self.lp)
        self.lit = [None] * n                # 0x300 coders per table, made on first use
        self.pos_slot = [[1024] * 64 for _ in range(4)]
        self.align = [1024] * 16
        self.pos_dec = [1024] * 115
        self.lens = [[1024] * (2 + 256 + 256) for _ in range(2)]     # choice, choice2, low[16][8], mid[16][8], high[256]
        self.ready = True

    def put(self, b):
        self.out.append(b)
        self.dict_end += 1
        if self.dict_end - self.dict_start == self.dict_size:
            self.dict_start += 1

    def put_all(self, bs):
        """put() of every byte of bs; the byte-by-byte dictStart rule runs where the gap can reach dictSize"""
        gap = self.dict_end - self.dict_start
        if gap + len(bs) < self.dict_size or gap >= self.dict_size or self.dict_size <= 0:
            self.out += bs
            self.dict_end += len(bs)
            return
        for b in bs:
            self.put(b)

    def copy(self, distance, length, strict=True):
        """`length` times put(byte(at: distance))"""
        if not 0 < distance <= self.dict_end:
            for _ in range(length):
                self.put(self.byte_at(distance, strict))
            return
        src = self.dict_end - distance
        if distance >= length:
            self.put_all(self.out[src:src + length])
        else:
            chunk = bytearray(length)
            for j in range(length):
                chunk[j] = self.out[src + j] if j < distance else chunk[j - distance]
            self.put_all(chunk)

    def byte_at(self, distance, strict=True):
        idx = self.dict_end - distance if distance <= self.dict_end else self.dict_size - distance + self.dict_end
        if not 0 <= idx < self.dict_end:
            if strict:
                raise Fail(TRAP)
            return 0
        return self.out[idx]

    def lit_table(self):
        prev = 0 if self.dict_end == self.dict_start else self.byte_at(1)
        t = swift_shl(self.dict_end & (swift_shl(1, self.lp) - 1), self.lc) + swift_shr(prev, 8 - self.lc)
        if not 0 <= t < len(self.lit):
            raise Fail(TRAP)
        if self.lit[t] is None:
            self.lit[t] = [1024] * 0x300
        return t

    # --- the symbol grammar, shared by both directions: `c` encodes `want` or decodes (want None) ---
    def tree(self, c, arr, base, nbits, want):
        m = 1
        for i in range(nbits):
            m = (m << 1) + c.bit(arr, base + m, None if want is None else (want >> (nbits - 1 - i)) & 1)
        return m - (1 << nbits)

    def tree_rev(self, c, arr, base, nbits, want):
        m, sym = 1, 0
        for i in range(nbits):
            b = c.bit(arr, base + m, None if want is None else (want >> i) & 1)
            m = (m << 1) + b
            sym |= b << i
        return sym

    def length(self, c, k, pos_state, want):
        """LZMALenDecoder.decode -> (zero-based length, branch); k 0 = match lengths, 1 = rep lengths"""
        L = self.lens[k]
        if pos_state >= 16:                  # 16 low / mid coders: the decoder traps, the writer codes bits nobody reads
            if want is None:
                raise Fail(TRAP)
            pos_state &= 15
        if c.bit(L, 0, None if want is None else int(want >= 8)) == 0:
            return self.tree(c, L, 2 + pos_state * 8, 3, want), "low"
        if c.bit(L, 1, None if want is None else int(want >= 16)) == 0:
            return 8 + self.tree(c, L, 130 + pos_state * 8, 3, None if want is None else want - 8), "mid"
        return 16 + self.tree(c, L, 258, 8, None if want is None else want - 16), "high"

    def literal(self, c, want):
        """-> (byte, table, bit at which a matched literal leaves the match byte, or None)"""
        t = self.lit_table()
        probs = self.lit[t]
        symbol, left = 1, None
        if self.state >= 7:
            match_byte = self.byte_at(self.reps[0] + 1, strict=want is None)
            k = 0
            while True:
                match_bit = (match_byte >> 7) & 1
                match_byte = (match_byte << 1) & 0xFF
                b = c.bit(probs, ((1 + match_bit) << 8) + symbol, None if want is None else (want >> (7 - k)) & 1)
                symbol = (symbol << 1) | b
                k += 1
                if match_bit != b:
                    left = k - 1
                    break
                if symbol >= 0x100:
                    break
        while symbol < 0x100:
            k = symbol.bit_length() - 1
            symbol = (symbol << 1) | c.bit(probs, symbol, None if want is None else (want >> (7 - k)) & 1)
        return symbol - 0x100, t, left

    def distance(self, c, length0, want):
        """pos slot and distance of a simple match -> (rep0, slot)"""
        len_state = min(length0, 3)
        slot = self.tree(c, self.pos_slot[len_state], 0, 6, None if want is None else pos_slot_of(want))
        if slot < 4:
            return slot, slot
        nd = (slot >> 1) - 1
        dist = (2 | (slot & 1)) << nd
        rem = None if want is None else want - dist
        if slot < 14:
            dist += self.tree_rev(c, self.pos_dec, dist - slot, nd, rem)
        else:
            dist += c.direct(nd - 4, None if rem is None else rem >> 4) << 4
            dist += self.tree_rev(c, self.align, 0, 4, None if rem is None else rem & 15)
        return dist, slot


def swift_shl(x, n):
    return x << n if n >= 0 else x >> -n


# ------------------------------------------------------------------------------------------------------------ writer
def lit(b):
    return ("lit", b)


def match(length, rep0):
    return ("match", length, rep0)


def rep(k, length):
    return ("rep", k, length)


SHORT = ("short",)


def lit_vs_match(k):
    """a literal equal to the match byte except at bit k from the top (None: equal to it)"""
    return ("mlit", k)


def end(length=2):
    return ("match", length, END_MARKER)


def encode_ops(m, ops, extra=0, first=None):
    """Range-code `ops` through model `m` (which keeps evolving, as the decoder's would) -> coded bytes.  Invalid operations
    are coded all the same; the bytes they would copy are read permissively so that the writer can go on."""
    c = RangeEncoder()
    if not m.ready:
        m.reset()                            # an LZMA2 chunk of reset kind 0 first: the decoder traps on it
    for op in ops:
        ps = m.dict_end & (swift_shl(1, m.pb) - 1)
        kind = op[0]
        if kind == "mlit":
            mb = m.byte_at(m.reps[0] + 1, strict=False)
            op = ("lit", mb if op[1] is None else mb ^ (0x80 >> op[1]))
            kind = "lit"
        c.bit(m.probs, (m.state << 4) + ps, int(kind != "lit"))
        if kind == "lit":
            b, _, _ = m.literal(c, op[1])
            m.put(b)
            m.state = 0 if m.state < 4 else m.state - 3 if m.state < 10 else m.state - 6
            continue
        c.bit(m.probs, 193 + m.state, int(kind != "match"))
        if kind == "match":
            length, rep0 = op[1], op[2]
            m.reps = [rep0] + m.reps[:3]
            m.length(c, 0, ps, length - 2)
            m.state = 7 if m.state < 7 else 10
            m.distance(c, min(length - 2, 3), rep0)
            if rep0 == END_MARKER:
                continue
        else:
            short = kind == "short"
            k = 0 if short else op[1]
            c.bit(m.probs, 205 + m.state, int(k != 0))
            if k == 0 and 241 + (m.state << 4) + ps < 432:       # (at 432 the decoder traps before reading it)
                c.bit(m.probs, 241 + (m.state << 4) + ps, int(not short))
            if k == 0:
                if short:
                    m.state = 9 if m.state < 7 else 11
                    m.put(m.byte_at(m.reps[0] + 1, strict=False))
                    continue
            else:
                c.bit(m.probs, 217 + m.state, int(k >= 2))
                if k >= 2:
                    c.bit(m.probs, 229 + m.state, int(k == 3))
                m.reps = [m.reps[k]] + m.reps[:k] + m.reps[k + 1:]
            length = op[2]
            m.length(c, 1, ps, length - 2)
            m.state = 8 if m.state < 7 else 11
        m.copy(m.reps[0] + 1, length, strict=False)
    data = bytearray(c.finish(extra))
    if first is not None:
        data[0] = first
    return bytes(data)


def write_lzma(ops, lc=3, lp=0, pb=2, dict_size=1 << 24, extra=0, first=None):
    """a raw LZMA stream (the properties are given separately, as LZMA.decompress(data:properties:) takes them)"""
    m = Model(lc, lp, pb, dict_size)
    m.reset()
    return encode_ops(m, ops, extra, first)


def props_byte(lc, lp, pb):
    return (pb * 5 + lp) * 9 + lc


def lzma_header(props, dict_size, usize):
    """the 13-byte .lzma header: properties byte, 4-byte dictionary size, 8-byte size (-1: unknown)"""
    return bytes([props]) + (dict_size & 0xFFFFFFFF).to_bytes(4, "little") + (usize & (1 << 64) - 1).to_bytes(8, "little")


class Stored:
    def __init__(self, payload, reset_dict=True, control=None, size=None):
        self.payload, self.reset_dict, self.control, self.size = bytes(payload), reset_dict, control, size


class Chunk:
    """an LZMA chunk: `reset` kind 0..3, `props` (lc, lp, pb) or a raw properties byte for kinds 2 and 3; unpack / comp
    override the declared sizes (None: the true ones), control overrides the whole control byte"""

    def __init__(self, ops, reset=0, props=None, unpack=None, comp=None, control=None, extra=0, first=None):
        self.ops, self.reset, self.props, self.unpack, self.comp = ops, reset, props, unpack, comp
        self.control, self.extra, self.first = control, extra, first


def write_lzma2(chunks, dict_size=1 << 20, end=True):
    """an LZMA2 stream (without its dictionary byte) from Stored / Chunk items; `end` appends the 0 control byte"""
    m = Model(dict_size=max(dict_size, 4096))
    out = bytearray()
    for ch in chunks:
        if isinstance(ch, Stored):
            if ch.reset_dict:
                m.dict_start = m.dict_end
            for b in ch.payload:
                m.put(b)
            n = (len(ch.payload) if ch.size is None else ch.size) - 1
            out += bytes([ch.control if ch.control is not None else 1 if ch.reset_dict else 2, n >> 8 & 0xFF, n & 0xFF])
            out += ch.payload
            continue
        pb_ = None
        if ch.reset >= 2:
            pb_ = ch.props if isinstance(ch.props, int) else props_byte(*(ch.props or (3, 0, 2)))
            if pb_ < 225:
                m.lc, m.pb, m.lp = pb_ % 9, pb_ // 45, (pb_ // 9) % 5
        if ch.reset >= 1:
            m.reset()
        if ch.reset == 3:
            m.dict_start = m.dict_end
        before = len(m.out)
        coded = encode_ops(m, ch.ops, ch.extra, ch.first)
        unpack = (len(m.out) - before if ch.unpack is None else ch.unpack) - 1
        comp = (len(coded) if ch.comp is None else ch.comp) - 1
        assert 0 <= unpack < 1 << 21 and 0 <= comp < 1 << 16, (unpack, comp)
        control = ch.control if ch.control is not None else 0x80 | ch.reset << 5 | unpack >> 16
        out += bytes([control, unpack >> 8 & 0xFF, unpack & 0xFF, comp >> 8, comp & 0xFF])
        if pb_ is not None:
            out.append(pb_)
        out += coded
    if end:
        out.append(0)
    return bytes(out)


def lzma2_dict_size(db):
    """LZMA2Decoder.init: None for a refused byte; the didSet clamp to 4096 applies"""
    if db & 0xC0 or (db & 0x3F) >= 40:
        return None
    bits = db & 0x3F
    return max((2 | (bits & 1)) << (bits // 2 + 11), 4096)


# ------------------------------------------------------------------------------------------------------------ decoder model
class Result:
    __slots__ = ("status", "out", "consumed", "trace", "wide", "controls")

    def __init__(self, status, out, consumed, trace, wide=None, controls=()):
        self.status, self.out, self.consumed, self.trace, self.wide = status, bytes(out), consumed, trace, wide
        self.controls = list(controls)

    def batch_status(self):
        """what the batched entry points answer: UNSUPPORTED once a chunk with lc + lp > 4 starts decoding"""
        return UNSUPPORTED if self.wide is not None else self.status


def _decode(m, rd, usize):
    """LZMADecoder.decode() LZMADecoder.swift:107-284, recording one trace entry per symbol:
    (kind, state before, posState, detail) with detail the literal table and leaving bit, the rep length branch, or the
    (length branch, pos slot) of a match"""
    c = RangeDecoder(rd)
    if not m.ready:
        raise Fail(TRAP)                     # the empty probability arrays of an LZMA2 chunk of reset kind 0 before any reset
    if len(m.lit) > 16 and m.wide is None:
        m.wide = len(m.out)                  # the batched kernels keep 16 literal tables: they stop here
    tr = m.trace
    while True:
        if usize == 0 and c.code == 0:
            return usize
        ps = m.dict_end & (swift_shl(1, m.pb) - 1)
        st0 = m.state
        i = (m.state << 4) + ps
        if c.bit(m.probs, i) == 0:
            if usize == 0:
                raise Fail(EXCEEDED)
            b, t, left = m.literal(c, None)
            usize -= 1
            m.put(b)
            m.state = 0 if m.state < 4 else m.state - 3 if m.state < 10 else m.state - 6
            tr.append(("mlit" if st0 >= 7 else "lit", st0, ps, (t, left), m.chunk))
            continue
        if c.bit(m.probs, 193 + m.state) != 0:
            if usize == 0:
                raise Fail(EXCEEDED)
            if m.dict_end == m.dict_start:
                raise Fail(WINDOW_EMPTY)
            if c.bit(m.probs, 205 + m.state) == 0:
                j = 241 + (m.state << 4) + ps
                if j >= 432:
                    raise Fail(TRAP)
                if c.bit(m.probs, j) == 0:
                    m.state = 9 if m.state < 7 else 11
                    m.put(m.byte_at(m.reps[0] + 1))
                    usize -= 1
                    tr.append(("short", st0, ps, None, m.chunk))
                    continue
                k = 0
            else:
                if c.bit(m.probs, 217 + m.state) == 0:
                    k = 1
                else:
                    k = 2 if c.bit(m.probs, 229 + m.state) == 0 else 3
                m.reps = [m.reps[k]] + m.reps[:k] + m.reps[k + 1:]
            length, branch = m.length(c, 1, ps, None)
            m.state = 8 if m.state < 7 else 11
            tr.append((f"rep{k}", st0, ps, (branch, length), m.chunk))
        else:
            m.reps = [m.reps[0]] + m.reps[:3]
            length, branch = m.length(c, 0, ps, None)
            m.state = 7 if m.state < 7 else 10
            rep0, slot = m.distance(c, length, None)
            m.reps[0] = rep0
            if rep0 & 0xFFFFFFFF == END_MARKER:
                tr.append(("end", st0, ps, (branch, length, slot), m.chunk))
                if c.code != 0:
                    raise Fail(FINISH_ERROR)
                return usize
            tr.append(("match", st0, ps, (branch, length, slot, rep0), m.chunk))
            if usize == 0:
                raise Fail(EXCEEDED)
            if rep0 >= m.dict_size or (rep0 > m.dict_end and m.dict_end < m.dict_size):
                raise Fail(NOT_ENOUGH)
        length += 2
        if -1 < usize < length:
            raise Fail(REPEAT_EXCEED)
        d = m.reps[0] + 1
        if d > m.dict_end:
            m.byte_at(d)                     # the wrapped branch: dictSize - d + dictEnd is never below dictEnd here
            raise AssertionError("byte(at:) read a wrapped index in range")
        m.copy(d, length)
        usize -= length


def decode_lzma(data, lc, lp, pb, dict_size, usize=-1, start=0):
    """LZMA.decompress(data:properties:uncompressedSize:) on data[start:] -> Result (consumed counted from `start`)"""
    m = Model(lc, lp, pb, dict_size)
    rd = Reader(data, start)
    try:
        m.reset()
        _decode(m, rd, -1 if usize is None or usize < 0 else usize)
        st = OK
    except Fail as e:
        st = e.code
    return Result(st, m.out, rd.pos - start, m.trace, m.wide)


def decode_lzma_alone(data):
    """LZMA.decompress(data:) LZMA.swift:25-34"""
    if len(data) < 13:
        return Result(WRONG_PROPERTIES, b"", 0, [])
    b = data[0]
    if b >= 225:
        return Result(WRONG_PROPERTIES, b"", 0, [])
    ds = int.from_bytes(data[1:5], "little")
    us = int.from_bytes(data[5:13], "little", signed=True)
    r = decode_lzma(data, b % 9, (b // 9) % 5, b // 45, ds, us, start=13)
    r.consumed += 13
    return r


def decode_lzma2(data, dict_byte):
    """LZMA2Decoder (LZMA2Decoder.swift:17-99) on data, the dictionary byte given apart -> Result"""
    ds = lzma2_dict_size(dict_byte)
    if ds is None:
        return Result(WRONG_DICT, b"", 0, [])
    m = Model(dict_size=ds)
    rd = Reader(data)
    st = OK
    try:
        while True:
            m.controls.append(rd.pos)
            control = rd.byte()
            if control == 0:
                break
            if control in (1, 2):
                if control == 1:
                    m.dict_start = m.dict_end
                size = (rd.byte() << 8) + rd.byte() + 1
                if rd.left() < size:
                    raise Fail(TRAP)
                for _ in range(size):
                    m.put(rd.byte())
                continue
            if control < 0x80:
                raise Fail(WRONG_CONTROL)
            m.chunk = rd.pos - 1
            reset = (control & 0x60) >> 5
            unpack = ((control & 0x1F) << 16) + (rd.byte() << 8) + rd.byte() + 1
            comp = (rd.byte() << 8) + rd.byte() + 1
            if reset == 1:
                m.reset()
            elif reset >= 2:
                b = rd.byte()
                if b >= 225:
                    raise Fail(WRONG_PROPERTIES)
                m.lc, m.pb, m.lp = b % 9, b // 45, (b // 9) % 5
                m.reset()
                if reset == 3:
                    m.dict_start = m.dict_end
            out0, in0 = len(m.out), rd.pos
            _decode(m, rd, unpack)
            if not (unpack == len(m.out) - out0 and rd.pos - in0 == comp):
                raise Fail(WRONG_SIZES)
    except Fail as e:
        st = e.code
    return Result(st, m.out, rd.pos, m.trace, m.wide, m.controls)
