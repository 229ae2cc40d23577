"""A catalogue of LZ4 streams as units of the batched frame decoder (swc_lz4_frame_decompress_batch), written with
tests/lz4_writer.py.  Each case carries the dictionary and dictionary ID it is decoded with and the reference's answer from
the writer's model of LZ4.decompress(data:dictionary:dictionaryID:): status, bytes, consumed bytes.  `kind` / `n_blocks` are
what the writer knows of the frame (None where the case was not laid out block by block)."""
import struct

import helpers as H
import lz4_cases as LC
import lz4_writer as W
from lz4_writer import FBlock

PAYLOAD = (W.OK, W.CHECKSUM)
NONE, INDEPENDENT, DEPENDENT, LEGACY = 0, 1, 2, 3
DICT = LC.dictionary(4096)


class FCase:
    def __init__(self, name, data, dictionary=None, dict_id=None, kind=None, n_blocks=None):
        self.name, self.data, self.dictionary, self.dict_id = name, bytes(data), dictionary, dict_id
        self.kind, self.n_blocks = kind, n_blocks
        self.model = W.decode(self.data, dictionary, dict_id)
        self.status, self.out = self.model.status, self.model.out
        self.consumed = self.model.next if self.status in PAYLOAD else 0

    @property
    def key(self):
        return (self.dictionary, self.dict_id)


def skippable(payload=b"abc", magic=0x184D2A50, size=None):
    return struct.pack("<II", magic, len(payload) if size is None else size) + payload


def cblock(j, prefix=0):
    """a small compressed block: three literals, a match of nine at offset 3 (or `prefix` bytes back), twelve literals"""
    return W.block([(LC.rb(3, 5900 + j), 9, prefix or 3)], LC.rb(12, 6000 + j))


def mixed_blocks(nb):
    """nb blocks: compressed, stored and empty stored ones in turn"""
    out = []
    for j in range(nb):
        out.append(FBlock(b"", stored=True) if j % 7 == 3 else FBlock(LC.rb(5 + j % 40, 7100 + j), stored=True) if j % 3 == 1
                   else FBlock(cblock(j)))
    return out


def existing_material():
    cases = []
    for c in LC.catalogue():
        if c.form == "frame":
            cases.append(FCase("family8 " + c.name, c.data, c.dictionary))
        for form, stream, d in LC.wrapped(c):
            kind = {"dependent": DEPENDENT, "independent": INDEPENDENT, "legacy": LEGACY}[form]
            # an empty block's mark is the EndMark; a legacy frame has no such mark
            cases.append(FCase(f"{form} {c.name}", stream, d, kind=kind, n_blocks=1 if c.data or kind == LEGACY else 0))
    from test_framing_handmade import LZ
    for name, blob, _ in LZ:
        cases.append(FCase("framing " + name, blob))
    small = H.fixture("LZ4/lz4_small_dict")
    for rel, _ in H.fixtures("LZ4/"):
        if rel.endswith(".lz4") and len(H.fixture(rel)) < (4 << 20):
            cases.append(FCase("golden " + rel, H.fixture(rel)))
            cases.append(FCase("golden+dict " + rel, H.fixture(rel), small))
    return cases


def skippables():
    dep = W.frame([FBlock(cblock(0))])
    needs_dict = W.frame([FBlock(W.block([(b"", 8, 100)], LC.rb(12, 1)))])
    with_id = W.frame([FBlock(cblock(0))], dict_id=7)
    cases = [FCase("skip one", skippable() + dep, kind=DEPENDENT, n_blocks=1),
             FCase("skip several", skippable() + skippable(b"", 0x184D2A5F) + skippable(b"x" * 40, 0x184D2A57) + dep, DICT),
             FCase("skip size past unit", skippable(b"abc", size=4) + dep),
             FCase("skip size field cut", struct.pack("<I", 0x184D2A50) + b"\x01\x00"),
             FCase("skip huge size", skippable(b"", size=0xFFFFFFFF)),
             FCase("needs dict", needs_dict, DICT, kind=DEPENDENT, n_blocks=1),
             FCase("skip then needs dict", skippable() + needs_dict, DICT),
             FCase("needs dict independent", W.frame([FBlock(W.block([(b"", 8, 100)], LC.rb(12, 1)))], independent=True), DICT),
             FCase("skip then needs dict independent", skippable() + W.frame([FBlock(W.block([(b"", 8, 100)], LC.rb(12, 1)))], independent=True), DICT),
             FCase("dict id matches", with_id, DICT, 7), FCase("dict id differs", with_id, DICT, 8),
             FCase("dict id not asked", with_id, DICT), FCase("dict id no dict", with_id, None, 7),
             FCase("skip then dict id", skippable() + with_id, DICT, 7),
             FCase("skip then id mismatch dropped", skippable() + dep, DICT, 8),
             FCase("skip then under 4 bytes", skippable() + b"\x04\x22\x4D"),
             FCase("skip then nothing", skippable()),
             FCase("skip then legacy", skippable() + W.legacy_frame([cblock(1)]), DICT),
             FCase("unknown magic", b"\x05\x22\x4D\x18" + dep[4:]), FCase("empty", b""), FCase("three bytes", b"\x04\x22\x4D")]
    return cases


def block_counts():
    cases = []
    for nb in (0, 1, 31, 32, 33, 64, 65, 1000):
        for independent in (True, False):
            kind = INDEPENDENT if independent else DEPENDENT
            tag = f"{'ind' if independent else 'dep'} {nb} blocks"
            blocks = mixed_blocks(nb)
            cases.append(FCase(tag, W.frame(blocks, independent=independent), kind=kind, n_blocks=nb))
            if nb in (0, 33, 65):
                want = W.decode(W.frame(blocks, independent=independent)).out
                cases.append(FCase(tag + " all flags", W.frame(blocks, independent=independent, block_checksums=True,
                                                               content_size=len(want), content_checksum=want, bd=0x40),
                                   kind=kind, n_blocks=nb))
                cases.append(FCase(tag + " dict", W.frame(blocks, independent=independent), DICT, kind=kind, n_blocks=nb))
    for bd, size in W.BLOCK_SIZES.items():
        full = LC.rb(97, bd) * (size // 97 + 1)
        for independent in (True, False):
            for extra in (0, 1):
                blocks = [FBlock(cblock(1)), FBlock(full[:size + extra], stored=True), FBlock(cblock(2))]
                cases.append(FCase(f"bd {bd:#x} stored block of max{'+1' if extra else ''} {'ind' if independent else 'dep'}",
                                   W.frame(blocks, independent=independent, bd=bd),
                                   kind=INDEPENDENT if independent else DEPENDENT, n_blocks=1 + (1 - extra) * 2))
    return cases


def error_order():
    """block k fails (its last literals cut), a bad checksum on k - 1 / k / k + 1, for independent frames (lz4_cases.chains()
    has the grid for dependent ones); a framing error at block k behind a failing or a sound block k - 1"""
    cases = []
    for nb in (1, 2, 33, 65):
        for k in sorted({0, nb // 2, 31 if nb > 32 else 0, 32 if nb > 32 else 0, nb - 1}):
            for bad in (None, k - 1, k, k + 1):
                if bad is not None and not 0 <= bad < nb:
                    continue
                blocks = [FBlock(cblock(j)[:-3] if j == k else cblock(j), ck=(0x12345678 if j == bad else None)) for j in range(nb)]
                tag = "none" if bad is None else f"{bad - k:+d}"
                cases.append(FCase(f"ind_{nb}_fail_{k}_badck_{tag}", W.frame(blocks, independent=True, block_checksums=True),
                                   kind=INDEPENDENT))
    for independent in (True, False):
        for prev_fails in (False, True):
            for nb in (1, 2, 33):
                good = [FBlock(cblock(j)) for j in range(nb - 1)]
                prev = [FBlock(cblock(99)[:-3] if prev_fails else cblock(99))]
                tag = f"{'ind' if independent else 'dep'} {nb}+1 {'failing' if prev_fails else 'sound'} k-1"
                kw = dict(independent=independent, bd=0x40)
                cases.append(FCase(tag + " size > max", W.frame(good + prev + [FBlock(b"", size=65537)], end=False, **kw)))
                whole = W.frame(good + prev + [FBlock(cblock(5))], **kw)
                cases.append(FCase(tag + " cut mark", whole[:len(W.frame(good + prev, end=False, **kw)) + 2]))
                cases.append(FCase(tag + " block past unit", whole[:-6]))
                ck = W.frame(good + prev + [FBlock(cblock(5))], block_checksums=True, **kw)
                cases.append(FCase(tag + " room for checksum missing", ck[:-5]))       # size + 4 present, not the checksum's 4
    return cases


def content_fields():
    cases = []
    for independent in (True, False):
        for blocks in ([], mixed_blocks(5)):
            want = W.decode(W.frame(blocks, independent=independent)).out
            tag = f"{'ind' if independent else 'dep'} {len(blocks)} blocks "
            f = lambda **kw: W.frame(blocks, independent=independent, **kw)
            cases += [FCase(tag + "size right", f(content_size=len(want))), FCase(tag + "size wrong", f(content_size=len(want) + 1)),
                      FCase(tag + "size > Int.max", f(content_size=1 << 63)),
                      FCase(tag + "checksum right", f(content_checksum=want)), FCase(tag + "checksum wrong", f(content_checksum=want + b"x")),
                      FCase(tag + "checksum missing", f(content_checksum=want)[:-4]),
                      FCase(tag + "checksum cut", f(content_checksum=want)[:-1]),
                      FCase(tag + "size wrong, checksum missing", f(content_size=len(want) + 1, content_checksum=want)[:-4]),
                      FCase(tag + "size wrong, checksum wrong", f(content_size=len(want) + 1, content_checksum=1))]
    return cases


def legacy():
    blocks = [cblock(j) for j in range(3)]
    whole = W.legacy_frame(blocks)
    cases = [FCase("legacy end of unit", whole, kind=LEGACY, n_blocks=3), FCase("legacy no blocks", W.legacy_frame([]), kind=LEGACY, n_blocks=0),
             FCase("legacy 40 blocks", W.legacy_frame([cblock(j) for j in range(40)]), DICT, kind=LEGACY, n_blocks=40)]
    for name, magic in (("frame", W.FRAME_MAGIC), ("legacy", W.LEGACY_MAGIC), ("skippable", 0x184D2A53)):
        cases.append(FCase(f"legacy ended by {name} magic", whole + struct.pack("<I", magic) + b"rest", kind=LEGACY, n_blocks=3))
    cases += [FCase("legacy cut size field", whole + b"\x10\x00"), FCase("legacy zero-size block", whole + struct.pack("<I", 0) + blocks[0]),
              FCase("legacy block past unit", whole[:-1]), FCase("legacy bad block", W.legacy_frame([blocks[0], blocks[1][:-3], blocks[2]])),
              FCase("legacy needs dict", W.legacy_frame([W.block([(b"", 8, 100)], LC.rb(12, 1))]), DICT)]
    return cases


def trailing():
    first = W.frame(mixed_blocks(4), independent=True, content_checksum=W.decode(W.frame(mixed_blocks(4), independent=True)).out)
    second = W.frame([FBlock(cblock(9))])
    return [FCase("trailing bytes", first + b"\x00\x01\x02garbage"), FCase("second frame behind", first + second),
            FCase("second frame behind dependent", second + first, DICT), FCase("second frame cut", second + first[:9])]


_CAT = None


def catalogue():
    global _CAT
    if _CAT is None:
        _CAT = existing_material() + skippables() + block_counts() + error_order() + content_fields() + legacy() + trailing()
        names = [c.name for c in _CAT]
        assert len(set(names)) == len(names), [n for n in names if names.count(n) > 1][:5]
    return _CAT


def truncations(limit=400):
    """every proper prefix of every case of at most `limit` bytes, the rest of the stream behind it -> [(FCase, tail)]"""
    out = []
    for c in catalogue():
        if len(c.data) <= limit:
            for k in range(len(c.data)):
                out.append((FCase(f"{c.name}[:{k}]", c.data[:k], c.dictionary, c.dict_id), c.data[k:]))
    return out
