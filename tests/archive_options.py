"""GzipArchive.archive option sets for the archive batch tests: each as the keywords of api.GzipArchive.archive and as
those of the CPU restatement (oracle/swco_deflatec.gzip_archive)."""
import itertools
import random

OS_BYTES = {"fat": 0, "unix": 3, "macintosh": 7, "ntfs": 11, "other": 255, None: 255}
COMMENTS = (None, "", "comment \xe9", "z\0", "\0")
NAMES = (None, "", "file.txt", "name\0")
MTIMES = (None, 0, -1.5, -7, 1700000000.75, 2**32, 2**32 + 5, 2**40 + 5)


def extra_sets():
    """0-3 extra fields, up to an XLEN of exactly 65 535"""
    from swcompression_b200 import ExtraField as E
    return [[], [E(65, 66, b"")], [E(1, 2, b"xy"), E(3, 4, bytes(300))],
            [E(5, 6, b"a"), E(7, 8, b""), E(9, 10, bytes(range(256)) * 3)], [E(1, 1, bytes(65531))],
            [E(2, 3, bytes(30000)), E(4, 5, bytes(35527))]]


def grid(seed=2):
    """-> [(archive keywords, oracle keywords)]: every comment x name x FHCRC x OS byte, with mtime, text flag and extra
    fields drawn in turn"""
    rng = random.Random(seed)
    extras = extra_sets()
    out = []
    for k, (comment, name, hcrc, os) in enumerate(itertools.product(COMMENTS, NAMES, (False, True), OS_BYTES)):
        mt = MTIMES[k % len(MTIMES)]
        ex = extras[k % len(extras)]
        tx = rng.random() < 0.5
        api = dict(comment=comment, fileName=name, writeHeaderCRC=hcrc, isTextFile=tx, osType=os, modificationTime=mt,
                   extraFields=ex)
        out.append((api, oracle_keywords(api)))
    return out


def oracle_keywords(api):
    mt, c, f = api.get("modificationTime"), api.get("comment"), api.get("fileName")
    return dict(comment=None if c is None else c.encode("latin-1"), fileName=None if f is None else f.encode("latin-1"),
                writeHeaderCRC=api.get("writeHeaderCRC", False), isTextFile=api.get("isTextFile", False),
                osByte=OS_BYTES[api.get("osType")], modificationTime=None if mt is None else int(mt),
                extraFields=[(e.si1, e.si2, bytes(e.bytes)) for e in api.get("extraFields", ())])
