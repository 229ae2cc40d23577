#!/usr/bin/env python3
"""Single-stream latency through the Swift-mirror API (the shape of the reference's own `swcomp benchmark run un-gzip / un-bz2 /
un-xz / lz4` rows: ONE archive, host memory in, host memory out), plus a zlib row and a 256 MiB stored gzip member, where the
single call is nearly a copy plus its CRC-32.  Prints MB/s of decompressed output and compressed input.

    python tools/bench_single.py [MiB, default 16] [row-name prefixes, comma-separated, default all]"""
import bz2
import gzip
import json
import lzma
import os
import sys
import time
import zlib

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
sys.path.insert(0, os.path.join(ROOT, "oracle"))
import helpers as H  # noqa: E402


def best(fn, arg, reps=3):
    fn(arg)
    ts = []
    out = None
    for _ in range(reps):
        t = time.perf_counter()
        out = fn(arg)
        ts.append(time.perf_counter() - t)
    return min(ts), out


def main():
    import swco
    from swcompression_b200 import BZip2, GzipArchive, LZ4, XZArchive, ZlibArchive
    mib = int(sys.argv[1]) if len(sys.argv) > 1 else 16
    only = sys.argv[2].split(",") if len(sys.argv) > 2 else None      # e.g. "gzip,zlib": the rows whose name starts so
    raw = b"".join(H.textlike(1 << 20, 7000 + i) for i in range(mib))
    blocks = [raw[i:i + (4 << 20)] for i in range(0, len(raw), 4 << 20)]
    stored = lambda: np.random.default_rng(7000).integers(0, 256, 256 << 20, dtype=np.uint8).tobytes()
    cases = [   # (name, decompressed bytes, compress, GPU call, CPU port)
        ("gzip (Deflate, 1 member)", lambda: raw, lambda r: gzip.compress(r, 6), GzipArchive.unarchive, swco.gzip_unarchive),
        ("zlib (Deflate, 1 stream)", lambda: raw, lambda r: zlib.compress(r, 6), ZlibArchive.unarchive, swco.zlib_unarchive),
        ("gzip level 0 (stored, 256 MiB)", stored, lambda r: gzip.compress(r, 0), GzipArchive.unarchive, swco.gzip_unarchive),
        ("bzip2 -9 (%d blocks)" % ((len(raw) + 899999) // 900000), lambda: raw, lambda r: bz2.compress(r, 9), BZip2.decompress,
         swco.bzip2_decompress),
        ("xz -6 (1 block)", lambda: raw, lambda r: lzma.compress(r, preset=6), XZArchive.unarchive, swco.xz_unarchive),
        ("lz4 frame, independent 4 MiB blocks", lambda: raw, lambda r: H.lz4_frame_independent(blocks, bd=0x70), LZ4.decompress,
         swco.lz4_decompress),
    ]
    for name, data, compress, fn, ofn in cases:
        if only and not any(name.startswith(o) for o in only):
            continue
        want = data()
        comp = compress(want)
        dt, out = best(fn, comp)
        assert out == want, name
        t = time.perf_counter()
        ost, oout, _ = ofn(comp)
        cdt = time.perf_counter() - t
        assert ost == 0 and oout == want
        print(json.dumps({"case": name, "raw_MiB": len(want) >> 20, "compressed_bytes": len(comp), "gpu_ms": dt * 1e3,
                          "gpu_out_MBps": len(want) / dt / 1e6, "gpu_in_MBps": len(comp) / dt / 1e6,
                          "cpu_port_1thread_out_MBps": len(want) / cdt / 1e6}))


if __name__ == "__main__":
    main()
